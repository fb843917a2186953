"""CPU checks for tests/test_gpu_attention_parity.py: the float64 closed forms of oracle/attn_ref.py equal float64
autograd of the reference's expressions, the GPU case table reaches every class it lists, and the per-element bounds
have teeth.

The location-aware step is emulated in float32 with the kernels' arithmetic: the CS-way time split of the energies and
the backward, the E/CS feature split of the context and of d(attn) with their lane / warp-tree orders, 32-frame
backward tiles, the per-CTA partials (d(q), weight gradients) summed over the cluster afterwards, and the decode loop's
accumulators.  The correct emulation must sit well inside the bounds; each of eight defects a kernel could plausibly
have must exceed them.
"""

import numpy as np
import pytest
import torch

import test_gpu_attention_parity as G
from oracle import attn_ref as ar

F32 = np.float32


# ------------------------------------------------------------------------------------------- oracle pin
def test_oracle_matches_float64_autograd_of_the_reference():
    from test_gpu_dot_attention import _dot_attention_torch
    from test_gpu_kernel_variants import _loc_attention_torch
    g = torch.Generator().manual_seed(0)
    B, T, D, E, K, R, N, temp = 3, 13, 7, 8, 3, 2, 2, 0.7
    mk = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    lens = torch.tensor([13, 5, 1])
    x = [t.requires_grad_(True) for t in (mk(B, D), mk(B, T, D), mk(B, T, E), torch.rand(B, T, generator=g,
                                          dtype=torch.float64), mk(K, 1, 2 * R + 1), mk(D, K), mk(1, D), mk(1))]
    gc, ga = mk(B, E), mk(B, T)
    c, a = _loc_attention_torch(x[0], x[1], x[2], x[3], lens, *x[4:], temp)
    ((c * gc).sum() + (a * ga).sum()).backward()
    n = lambda t: t.detach().numpy()
    st = ar.loc_step(*(n(t) for t in x[:4]), lens.numpy(), n(x[4])[:, 0], n(x[5]), n(x[6])[0], n(x[7]), temp,
                     dctx=n(gc), dattn=n(ga))
    close = lambda got, ref: np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-12)
    close(st.attn, n(a))
    close(st.ctx, n(c))
    for got, leaf in ((st.dq, 0), (st.dkey, 1), (st.dvalue, 2), (st.dprev, 3), (st.dwc.sum(0)[:, None], 4),
                      (st.dwp.sum(0), 5), (st.dwe.sum(0)[None], 6), (st.dbe.sum(0)[None], 7)):
        close(got, n(x[leaf].grad))
    xd = [t.requires_grad_(True) for t in (mk(B * N, D), mk(B * N, T, D), mk(B * N, T, E))]
    gc, ga = mk(B * N, E), mk(B * N, T)
    c, a = _dot_attention_torch(*xd, lens, N, temp)
    ((c * gc).sum() + (a * ga).sum()).backward()
    st = ar.dot_step(*(n(t) for t in xd), lens.numpy(), N, temp, dctx=n(gc), dattn=n(ga))
    for got, ref in ((st.attn, a), (st.ctx, c), (st.dq, xd[0].grad), (st.dkey, xd[1].grad), (st.dvalue, xd[2].grad)):
        close(got, n(ref))


def test_cluster_rule_matches_the_library(pkg):
    lib = pkg.load_library()
    for T in (1, 7, 8, 15, 16, 31, 32, 149, 8192):
        for E in (4, 8, 64, 1024, 2048, 2064, 4092, 4096, 4100, 8192):
            assert lib.b200asr_locattn_cluster_size(T, E) == ar.cluster_size(T, E), (T, E)
            if E % 16 == 0 and E <= 4096:         # the backward's 1024-column limit holds for every T
                assert E // ar.cluster_size(T, E) <= 1024, (T, E)


# ------------------------------------------------------------------------------------------- coverage
def test_gpu_cases_reach_every_class(pkg):
    """Each case reaches a class no other case reaches (deleting any case fails here), and together with the limit
    and d(value) tests they reach every listed class."""
    lib = pkg.load_library()
    reached = {n: G.case_classes(lib, n) for n in G.CASES}
    reached.update({n: G.dvalue_classes(n) for n in G.DVALUE})
    reached.update({"limit " + f: c for f, c in G.LIMITS.items()})
    missing = G.REQUIRED_CLASSES - set().union(*reached.values())
    assert not missing, missing
    for name, r in reached.items():
        others = set().union(*(x for n, x in reached.items() if n != name))
        assert r - others, name
    # the limit test's memory length is the last one whose shared memory fits the H100's 227 KiB opt-in
    T = G.loc_bwd_longest_t(232448)
    assert G.loc_bwd_smem(T, 300, 2048, 10, 100) <= 232448 < G.loc_bwd_smem(T + 1, 300, 2048, 10, 100)


# ------------------------------------------------------------------------------------------- fp32 emulation
def fma(a, b, c):
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F32)


def tree(x):
    """xor-butterfly sum over the last axis (a power of two)."""
    while x.shape[-1] > 1:
        h = x.shape[-1] // 2
        x = (x[..., :h] + x[..., h:]).astype(F32)
    return x[..., 0]


def lanes(x, width=32):
    """[..., n] -> [..., ceil(n / width), width] zero-padded: element lane + width * i."""
    n = x.shape[-1]
    m = -(-n // width) * width
    x = np.concatenate([x, np.zeros(x.shape[:-1] + (m - n,), F32)], -1)
    return x.reshape(x.shape[:-1] + (m // width, width))


def lane_sum(prod_fn, n, shape):
    """per-lane fmaf chains over elements lane + 32 i, then a warp tree; prod_fn(i) -> (a, b) of chunk i [..., 32]."""
    acc = np.zeros(shape + (32,), F32)
    for i in range(-(-n // 32)):
        a, b = prod_fn(i)
        acc = fma(a, b, acc)
    return tree(acc)


class Case:
    def __init__(self, pkg, name, seed=1):
        lib = pkg.load_library()
        self.name = name
        fam, _, self.T, self.D, self.E, self.K, self.R, self.temp, _, _, _ = G.CASES[name]
        inp = G.make_inputs(lib, name, seed)
        self.B = inp["q"].shape[0]
        self.CS = lib.b200asr_locattn_cluster_size(self.T, self.E)
        self.inp = {k: v.numpy().astype(F32) if v.dtype == torch.float32 else v.numpy() for k, v in inp.items()}
        self.len = np.clip(self.inp["lens"], 0, self.T)


def emulate_fwd(c, prev, q, defect=None):
    B, T, D, E, K, R, CS = c.B, c.T, c.D, c.E, c.K, c.R, c.CS
    W = 2 * R + 1
    x = c.inp
    P = np.pad(prev, ((0, 0), (R, R + 1)))
    sh = 1 if defect == "conv shifted one frame" else 0
    conv = np.zeros((B, K, T), F32)
    for j in range(W):
        conv = fma(x["w_conv"][None, :, j, None], P[:, None, j + sh:j + sh + T], conv)
    pre = np.zeros((B, T, D), F32)
    for k in range(K):
        pre = fma(x["w_proj"][None, None, :, k], conv[:, k, :, None], pre)
    loc = np.tanh(pre)
    s = np.tanh(((x["key"] + q[:, None, :]).astype(F32) + loc).astype(F32))
    we = lanes(x["w_e"])
    sl = lanes(s)
    esum = lane_sum(lambda i: (we[i], sl[:, :, i]), D, (B, T))
    e = (((esum + x["b_e"][0]).astype(F32)) / F32(c.temp)).astype(F32)
    t = np.arange(T)[None]
    read = t <= c.len[:, None] if defect == "mask at t <= len" else t < c.len[:, None]
    read &= t < T
    e = np.where(read, e, -np.inf).astype(F32)
    mx = e.max(1, keepdims=True)
    ex = np.where(read, np.exp((e - mx).astype(F32)), F32(0)).astype(F32)
    ssum = np.zeros((B, 512), F32)
    exl = lanes(ex, 512)
    for i in range(exl.shape[1]):
        ssum = (ssum + exl[:, i]).astype(F32)
    a = (ex / tree(ssum)[:, None]).astype(F32)
    ES = E // CS
    ngroups = 512 // min(ES // 4, 512)
    acc = np.zeros((B, ngroups, E), F32)
    v = np.where(read[:, :, None], x["value"], F32(0))
    for i in range(-(-T // ngroups)):
        tt = np.arange(i * ngroups, min((i + 1) * ngroups, T))
        g = tt - i * ngroups
        acc[:, g] = fma(np.where(read[:, tt, None], a[:, tt, None], F32(0)), v[:, tt], acc[:, g])
    ctx = acc[:, 0]
    for g in range(1, ngroups):
        ctx = (ctx + acc[:, g]).astype(F32)
    return a, ctx, conv, pre, loc, s


def emulate_bwd(c, prev, q, A, dctx, dattn, defect=None):
    """-> per-row dq_part [B, CS, D], dkey, dvalue, dprev, wpart [B, CS, P]."""
    B, T, D, E, K, R, CS = c.B, c.T, c.D, c.E, c.K, c.R, c.CS
    W, TS, ES = 2 * R + 1, -(-c.T // c.CS), c.E // c.CS
    x = c.inp
    _, _, conv, pre, loc, s = emulate_fwd(c, prev, q)
    t = np.arange(T)[None]
    valid = t < c.len[:, None]
    v = np.where(valid[:, :, None], x["value"], F32(0))
    parts = []
    for rr in range(CS):
        vs = v[:, :, rr * ES:(rr + 1) * ES].reshape(B, T, -1, 32, 4)             # [B, T, k, lane, component]
        dc = dctx[:, rr * ES:(rr + 1) * ES].reshape(B, 1, -1, 32, 4)
        acc = np.zeros((B, T, 32), F32)
        for k in range(vs.shape[2]):
            for comp in range(4):
                acc = fma(dc[:, :, k, :, comp], vs[:, :, k, :, comp], acc)
        parts.append(np.where(valid, tree(acc), F32(0)))
    g = dattn.astype(F32)
    for rr in range(CS):
        if defect == "one CTA's d(attn) partial dropped" and rr == CS - 1:
            continue
        g = (g + parts[rr]).astype(F32)
    nthr = max(128, -(-D // 32) * 32)
    dl = lanes(np.where(valid, A * g, F32(0)), nthr)            # fmaf(attn, g, dot) per thread, then the block tree
    dot = np.zeros((B, nthr), F32)
    for i in range(dl.shape[1]):
        ai = lanes(np.where(valid, A, F32(0)), nthr)[:, i]
        gi = lanes(np.where(valid, g, F32(0)), nthr)[:, i]
        dot = fma(ai, gi, dot)
    dot = tree(np.pad(dot, ((0, 0), (0, 512 - nthr))) if nthr < 512 else dot)[:, None]
    de = (A * (g - dot).astype(F32)).astype(F32)
    if defect != "temperature missing in the softmax backward":
        de = (de / F32(c.temp)).astype(F32)
    de = np.where(valid, de, F32(0))
    we = x["w_e"][None]
    dq_part = np.zeros((B, CS, D), F32)
    dew = np.zeros((B, CS, D), F32)
    deb = np.zeros((B, CS), F32)
    dpw = np.zeros((B, CS, D, K), F32)
    dkey = np.zeros((B, T, D), F32)
    dloc_all = np.zeros((B, T, D), F32)
    for tl in range(TS):
        for rr in range(CS):
            tt = rr * TS + tl
            if tt >= T:
                continue
            ok = (tt < c.len)[:, None]
            ss = s[:, tt]
            dpre = ((de[:, tt, None] * we).astype(F32) * (F32(1) - (ss * ss).astype(F32)).astype(F32)).astype(F32)
            dpre = np.where(ok, dpre, F32(0))
            dew[:, rr] = np.where(ok, fma(de[:, tt, None], ss, dew[:, rr]), dew[:, rr])
            dq_part[:, rr] = (dq_part[:, rr] + dpre).astype(F32)
            lc = loc[:, tt]
            dloc = np.where(ok, (dpre * (F32(1) - (lc * lc).astype(F32))).astype(F32), F32(0))
            dpw[:, rr] = np.where(ok[:, :, None], fma(dloc[:, :, None], conv[:, None, :, tt], dpw[:, rr]), dpw[:, rr])
            deb[:, rr] = np.where(ok[:, 0], (deb[:, rr] + de[:, tt]).astype(F32), deb[:, rr])
            dkey[:, tt] = dpre
            dloc_all[:, tt] = dloc
    wpl = lanes(x["w_proj"].T)                                                     # [K, i, lane]
    dll = lanes(dloc_all)                                                          # [B, T, i, lane]
    dconv = np.stack([lane_sum(lambda i: (dll[:, :, i], wpl[k, i]), D, (B, T)) for k in range(K)], 1)
    dconv = np.where(valid[:, None], dconv, F32(0))
    if defect == "d(w_conv) partial over padded frames":   # d(conv) of padded frames left from the previous tile
        stale = np.roll(dconv, G.ATT_TT, axis=2)
        tile_start = (t % TS) >= G.ATT_TT
        dconv_w = np.where((~valid & tile_start)[:, None], stale, dconv)
    else:
        dconv_w = dconv
    P = np.pad(prev, ((0, 0), (R, R)))
    dwc = np.zeros((B, CS, K, W), F32)
    for tl in range(TS):
        for rr in range(CS):
            tt = rr * TS + tl
            if tt >= T:
                continue
            use = tt < (T if defect == "d(w_conv) partial over padded frames" else c.len)
            win = np.stack([P[:, tt + j] for j in range(W)], 1)                   # [B, W]
            new = fma(dconv_w[:, :, tt, None], win[:, None, :], dwc[:, rr])
            dwc[:, rr] = np.where(np.asarray(use)[:, None, None] if np.ndim(use) else use, new, dwc[:, rr])
    dcp = np.pad(dconv, ((0, 0), (0, 0), (2 * R, 2 * R)))
    idx = np.arange(K * W)
    kk, jj = idx // W, idx % W
    wcl = lanes(x["w_conv"].reshape(-1))
    dprev = np.zeros((B, T), F32)
    for tp in range(T):
        terms = lanes(dcp[:, kk, tp - jj + 3 * R])                # d(conv) at time tp - j + R: [B, i, lane]
        dprev[:, tp] = lane_sum(lambda i: (terms[:, i], wcl[i]), K * W, (B,))
    dvalue = np.where(valid[:, :, None], (A[:, :, None] * dctx[:, None, :]).astype(F32), F32(0))
    wpart = np.concatenate([dpw.reshape(B, CS, -1), dwc.reshape(B, CS, -1), dew, deb[:, :, None]], 2)
    if defect == "dq_part of rank 0 only":
        dq_part[:, 1:] = 0
    return dq_part, dkey, dvalue, dprev, wpart


def _oracle(c, prev, q, A=None, dctx=None, dattn=None):
    x = {k: v.astype(np.float64) if v.dtype == F32 else v for k, v in c.inp.items()}
    kw = {} if dctx is None else dict(dctx=dctx, dattn=dattn, attn=A)
    return ar.loc_step(q, x["key"], x["value"], prev, x["lens"], x["w_conv"], x["w_proj"], x["w_e"], x["b_e"],
                       c.temp, **kw)


def step_ratios(c, defect=None, seed=0):
    """worst err / bound of every output of one emulated step."""
    x = c.inp
    A, ctx, *_ = emulate_fwd(c, x["prev"], x["q"], defect)
    st = _oracle(c, x["prev"], x["q"])
    r = {"attn": ar.worst_ratio(A, st.attn, np.where(st.valid, st.attn_b + G.TINY, 0.0)),
         "ctx": ar.worst_ratio(ctx, st.ctx, st.ctx_b)}
    A, *_ = emulate_fwd(c, x["prev"], x["q"])
    dq, dkey, dvalue, dprev, wpart = emulate_bwd(c, x["prev"], x["q"], A, x["dctx"], x["dattn"], defect)
    st = _oracle(c, x["prev"], x["q"], A.astype(np.float64), x["dctx"], x["dattn"])
    D, K, W, B = c.D, c.K, 2 * c.R + 1, c.B
    wp = wpart.astype(np.float64).sum(1)
    r.update(dq=ar.worst_ratio(dq.astype(np.float64).sum(1), st.dq, st.dq_b),
             dkey=ar.worst_ratio(dkey, st.dkey, st.dkey_b), dvalue=ar.worst_ratio(dvalue, st.dvalue, st.dvalue_b),
             dprev=ar.worst_ratio(dprev, st.dprev, st.dprev_b))
    o = 0
    for f, m in (("dwp", D * K), ("dwc", K * W), ("dwe", D), ("dbe", 1)):
        r[f] = ar.worst_ratio(wp[:, o:o + m], getattr(st, f).reshape(B, -1), getattr(st, f + "_b").reshape(B, -1))
        o += m
    return r


def loop_ratios(c, L, defect=None):
    """An L-step decode loop: d(key) and the weight partials accumulated per step, d(value) once after the loop."""
    g = np.random.default_rng(5)
    x = c.inp
    prev = x["prev"]
    dkey = np.zeros((c.B, c.T, c.D), F32)
    wacc = None
    steps, As, dctxs = [], [], []
    for l in range(L):
        q = g.standard_normal((c.B, c.D)).astype(F32)
        dctx = g.standard_normal((c.B, c.E)).astype(F32)
        dattn = g.standard_normal((c.B, c.T)).astype(F32)
        A, *_ = emulate_fwd(c, prev, q)
        _, dk, _, _, wpart = emulate_bwd(c, prev, q, A, dctx, dattn)
        valid = (np.arange(c.T)[None] < c.len[:, None])[:, :, None]
        dkey = np.where(valid, (dkey + dk).astype(F32), dkey)
        wacc = wpart if wacc is None or defect == "wpart overwritten instead of accumulated" else (wacc + wpart).astype(F32)
        steps.append(_oracle(c, prev.astype(np.float64), q.astype(np.float64), A.astype(np.float64), dctx, dattn))
        As.append(A)
        dctxs.append(dctx)
        prev = A
    n = L - 1 if defect == "last decode step missing from attn_dvalue" else L
    dv = np.zeros((c.B, c.T, c.E), F32)
    for l in range(n):
        dv = fma(As[l][:, :, None], dctxs[l][:, None, :], dv)
    r = {}
    val, bnd = ar.accumulate(0.0, *zip(*((s.dkey, s.dkey_b, s.dkey_abs) for s in steps)))
    r["dkey"] = ar.worst_ratio(dkey, val, bnd)
    ref, bnd = ar.dvalue(np.stack(As, 1).astype(np.float64), np.stack(dctxs, 1).astype(np.float64))
    r["dvalue"] = ar.worst_ratio(dv, ref, bnd)
    wp = wacc.astype(np.float64).sum(1)
    val, bnd = ar.accumulate(0.0, *zip(*((s.dwp, s.dwp_b, s.dwp_abs) for s in steps)))
    r["dwp"] = ar.worst_ratio(wp[:, :c.D * c.K], val.reshape(c.B, -1), bnd.reshape(c.B, -1))
    return r


EMULATED = ["loc_t31", "loc_t16", "loc_cfg_minb2"]


@pytest.fixture(scope="module")
def cases(pkg):
    return {n: Case(pkg, n) for n in EMULATED}


@pytest.mark.parametrize("name", EMULATED)
def test_fp32_emulation_sits_inside_the_bounds(cases, name):
    c = cases[name]
    r = step_ratios(c)
    print(name, {k: "%.3g" % v for k, v in r.items()})
    assert max(r.values()) <= 0.5, r


def test_fp32_decode_loop_sits_inside_the_bounds(cases):
    r = loop_ratios(cases["loc_t16"], 4)
    print({k: "%.3g" % v for k, v in r.items()})
    assert max(r.values()) <= 0.5, r


@pytest.mark.parametrize("defect,name,output", [
    ("conv shifted one frame", "loc_t31", "attn"),
    ("one CTA's d(attn) partial dropped", "loc_cfg_minb2", "dkey"),
    ("dq_part of rank 0 only", "loc_cfg_minb2", "dq"),
    ("mask at t <= len", "loc_t16", "ctx"),
    ("temperature missing in the softmax backward", "loc_t31", "dkey"),
    ("d(w_conv) partial over padded frames", "loc_cfg_minb2", "dwc"),
])
def test_step_bound_rejects_defects(cases, defect, name, output):
    r = step_ratios(cases[name], defect)
    print(defect, {k: "%.3g" % v for k, v in r.items()})
    assert r[output] >= 10, r


@pytest.mark.parametrize("defect,output", [("last decode step missing from attn_dvalue", "dvalue"),
                                           ("wpart overwritten instead of accumulated", "dwp")])
def test_decode_loop_bound_rejects_defects(cases, defect, output):
    r = loop_ratios(cases["loc_t16"], 4, defect)
    print(defect, {k: "%.3g" % v for k, v in r.items()})
    assert r[output] >= 10, r
