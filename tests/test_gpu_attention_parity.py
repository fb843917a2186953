"""Attention kernels per element against the float64 closed forms of oracle/attn_ref.py, through the C ABI.

Every case pins the variant it exists for (cluster size CS, backward MINB instance) through the library's queries, and
the case table reaches every class in REQUIRED_CLASSES (checked on the CPU by tests/test_host_attn_bounds.py).  Inputs:
NaN in every padded key and value frame (the kernels must never read them; the oracle zeroes them), a nonzero previous
alignment on every frame (the location convolution's halo reads past len), NaN in every output a non-accumulating
call must write, and a sentinel pattern in the accumulators of the _acc calls (frames t >= len must stay bit-identical).
Per element, |kernel - float64| <= the bound derived in oracle/attn_ref.py, fixed before any run; a zero bound (masked
frames) demands exact equality.  Two runs of every case are bit-identical.
"""
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import attn_ref as ar

pytestmark = pytest.mark.gpu
DEV = "cuda"
ATT_TT = 32                      # time tile of the location backward
DV_TT, DV_SMEM = 8, 48 * 1024    # attn_dvalue: frames per CTA, shared-memory limit of its [L][DV_TT] stage
DOT_MAX_T = 8192
TINY = 2.0 ** -126               # expf of an energy far below the maximum underflows: absolute error of an attention
CFG = dict(D=300, E=2048, K=10, R=100)   # the location attention of every config/b200/*.yaml (E: cfg C's value)
RATIOS = {}                      # worst error / bound per kernel output, written to $ATTN_RATIOS_JSON when set

# name -> (family, B, T, D, E, K, R, temperature, lens, N, flags).  B = "minb2": sm_count // CS + 1 rows, so that
# the CTAs outnumber the SMs.  lens: the first rows' lengths; the remaining rows take lengths from T down to 1.
CASES = {
    "loc_t1": ("loc", 3, 1, 31, 64, 1, 0, 1.0, [1, 1, 5], 1, ()),
    "loc_t7_e4096": ("loc", 3, 7, 512, 4096, 16, 5, 0.7, [7, 3, 2], 1, ("sat",)),
    "loc_t8_e2048": ("loc", 3, 8, 300, 2048, 10, 100, 0.5, [8, 4, 1], 1, ()),
    "loc_t15": ("loc", 2, 15, 300, 64, 10, 100, 0.5, [15, 9], 1, ()),
    "loc_t16": ("loc", 3, 16, 300, 256, 4, 5, 0.7, [16, 8, 30], 1, ()),
    "loc_t31": ("loc", 2, 31, 300, 256, 10, 100, 0.5, [31, 16], 1, ()),
    "loc_t32": ("loc", 3, 32, 64, 256, 4, 5, 0.5, [32, 8, 17], 1, ()),
    "loc_cfg_minb2": ("loc", "minb2", 149, 300, 2048, 10, 100, 0.5, [149, 149, 32, 38, 76, 1, 200], 1, ("spread",)),
    "loc_d384_minb2": ("loc", "minb2", 64, 384, 2048, 10, 100, 0.5, [64, 33], 1, ()),
    "loc_d385": ("loc", "minb2", 64, 385, 2048, 10, 100, 0.5, [64, 33], 1, ()),
    "loc_e516": ("loc", "minb2", 64, 300, 2064, 10, 100, 0.5, [64, 33], 1, ()),
    "loc_ctx_2pass": ("loc", 2, 40, 300, 4092, 10, 100, 0.5, [40, 21], 1, ("fwd_only",)),
    "dot_t1": ("dot", 2, 1, 1, 64, 0, 0, 1.0, [1, 3], 2, ()),
    "dot_t7_e2048": ("dot", 2, 7, 300, 2048, 0, 0, 0.7, [7, 4], 2, ("spread",)),
    "dot_cfg_minb2": ("dot", "minb2", 149, 300, 2048, 0, 0, 0.5, [149, 38, 1, 300], 1, ()),
    "dot_e516": ("dot", "minb2", 64, 300, 2064, 0, 0, 0.5, [64, 33], 1, ()),
}
# the longest memories the backwards take at the configs' shapes, and the first they refuse (see test_backward_limits)
LIMITS = {"loc": {"loc bwd longest T", "loc bwd first refused T"}, "dot": {"dot bwd longest T", "dot bwd first refused T"}}
# b200asr_attn_dvalue: (B, L, T, E, accumulate); L = None is the longest L its shared-memory stage takes
DVALUE = {"dv_l1": (3, 1, 13, 64, 0), "dv_l46_acc": (2, 46, 149, 2048, 1), "dv_lmax_acc": (2, None, 21, 128, 1)}

REQUIRED_CLASSES = {
    "loc CS=1", "loc CS=2", "loc CS=4", "dot CS=1", "dot CS=2", "dot CS=4",
    "T=1", "T=7", "T=8", "T=15", "T=16", "T=31", "T=32", "T mod CS != 0",
    "len=1", "len on a slice boundary", "len on an ATT_TT boundary", "len=T", "len>T",
    "loc MINB=1", "loc MINB=2", "dot MINB=1", "dot MINB=2", "loc D=384 MINB=2", "loc D=385 MINB=1",
    "loc E/CS=512 MINB=2", "loc E/CS=516 MINB=1", "dot E/CS=512 MINB=2", "dot E/CS=516 MINB=1",
    "loc E/CS=1024 CS=4", "loc E/CS=1024 CS=2", "dot E/CS=1024 CS=2",
    "D=1", "D=31", "D=300", "D=512", "K=1", "K=16", "R=0", "2R+1>T", "temp=0.5", "temp=1", "temp=0.7",
    "context 2 passes", "saturated tanh", "one-hot and uniform rows",
    "loc bwd longest T", "loc bwd first refused T", "dot bwd longest T", "dot bwd first refused T",
    "dvalue L=1", "dvalue L=46", "dvalue L=max", "dvalue acc=0", "dvalue acc=1", "dvalue T mod 8 != 0",
}


def rows_of(lib, name):
    fam, B, T, D, E, K, R, temp, lens, N, flags = CASES[name]
    if B == "minb2":
        B = lib.b200asr_device_sm_count() // lib.b200asr_locattn_cluster_size(T, E) + 1
    return B


def case_lens(lib, name):
    fam, B, T, D, E, K, R, temp, lens, N, flags = CASES[name]
    B = rows_of(lib, name)
    rest = np.linspace(T, 1, max(B - len(lens), 1)).round().astype(np.int64)
    return np.concatenate([np.asarray(lens, np.int64), rest])[:B]


def minb(lib, name):
    fam, _, T, D, E = CASES[name][:5]
    B, N = rows_of(lib, name), CASES[name][9]
    if "fwd_only" in CASES[name][10]:
        return None
    return lib.b200asr_debug_locattn_bwd_minb(B, T, D, E) if fam == "loc" else lib.b200asr_debug_dotattn_bwd_minb(
        B * N, T, E)


def case_classes(lib, name):
    """The classes a case reaches, from its shape and the library's dispatch queries."""
    fam, _, T, D, E, K, R, temp, _, N, flags = CASES[name]
    cs = lib.b200asr_locattn_cluster_size(T, E)
    mb = minb(lib, name)
    ts = (T + cs - 1) // cs
    out = {"%s CS=%d" % (fam, cs), "temp=%g" % temp}
    out |= {"T=%d" % T} if T in (1, 7, 8, 15, 16, 31, 32) else set()
    out |= {"T mod CS != 0"} if T % cs else set()
    out |= {"D=%d" % D} if D in (1, 31, 300, 512) else set()
    if mb is not None:
        out.add("%s MINB=%d" % (fam, mb))
        if fam == "loc" and D in (384, 385):
            out.add("loc D=%d MINB=%d" % (D, mb))
        if E // cs in (512, 516):
            out.add("%s E/CS=%d MINB=%d" % (fam, E // cs, mb))
        if E // cs == 1024:
            out.add("%s E/CS=1024 CS=%d" % (fam, cs))
    if fam == "loc":
        out |= {"K=%d" % K} if K in (1, 16) else set()
        out |= {"R=0"} if R == 0 else set()
        out |= {"2R+1>T"} if 2 * R + 1 > T else set()
    if E // cs // 4 > 512:
        out.add("context 2 passes" if E // cs // 4 <= 1024 else "context 3+ passes")
    for ln in case_lens(lib, name):
        out |= {"len=1"} if ln == 1 else set()
        out |= {"len=T"} if ln == T else set()
        out |= {"len>T"} if ln > T else set()
        out |= {"len on a slice boundary"} if 0 < ln < T and cs > 1 and ln % ts == 0 else set()
        out |= {"len on an ATT_TT boundary"} if fam == "loc" and ts > ATT_TT and ln % ts == ATT_TT else set()
    out |= {"saturated tanh"} if "sat" in flags else set()
    out |= {"one-hot and uniform rows"} if "spread" in flags else set()
    return out


def dvalue_l(L):
    return DV_SMEM // (DV_TT * 4) if L is None else L


def dvalue_classes(name):
    B, L, T, E, acc = DVALUE[name]
    L = dvalue_l(L)
    out = {"dvalue acc=%d" % acc}
    out |= {"dvalue L=%d" % L} if L in (1, 46) else set()
    out |= {"dvalue L=max"} if L == dvalue_l(None) else set()
    out |= {"dvalue T mod 8 != 0"} if T % DV_TT else set()
    return out


def loc_bwd_smem(T, D, E, K, R):
    """Dynamic + static shared memory of b200asr_locattn_bwd(_acc)."""
    W, cs = 2 * R + 1, ar.cluster_size(T, E)
    return 4 * (T + 2 * R + K * W + D * K + 2 * D + 2 * T + cs * T + K * ATT_TT + ATT_TT * D + K * (T + 2 * R)) + 128


def loc_bwd_longest_t(optin):
    T = 1
    while loc_bwd_smem(T + 1, CFG["D"], CFG["E"], CFG["K"], CFG["R"]) <= optin:
        T += 1
    return T


# ------------------------------------------------------------------------------------------- inputs
def make_inputs(lib, name, seed):
    """float32 host tensors of a case; NaN in padded key / value frames."""
    fam, _, T, D, E, K, R, temp, _, N, flags = CASES[name]
    B = rows_of(lib, name)
    rows = B * N
    lens = torch.from_numpy(case_lens(lib, name))
    g = torch.Generator().manual_seed(seed)
    mk = lambda *s, sc=1.0: torch.randn(*s, generator=g) * sc
    inp = dict(lens=lens, q=mk(rows, D), key=mk(rows, T, D), value=mk(rows, T, E), dctx=mk(rows, E),
               dattn=mk(rows, T))
    if fam == "loc":
        W = 2 * R + 1
        inp.update(prev=torch.rand(B, T, generator=g) / T, w_conv=mk(K, W, sc=0.3), w_proj=mk(D, K, sc=0.5),
                   w_e=mk(D, sc=0.3), b_e=mk(1))
        if "sat" in flags or "spread" in flags:
            sgn = torch.sign(inp["w_e"])
            inp["key"][0, min(2, T - 1)] = 30 * sgn           # row 0: one saturated frame far above the others
            inp["key"][1] = -30 * sgn                          # row 1: every frame saturated alike: uniform
            inp["w_e"] *= 0.2
    else:
        if "spread" in flags:
            t0 = min(2, T - 1)                                 # row 0: q along key frame t0 (near one-hot)
            inp["q"][0] = 8 * inp["key"][0, t0] / inp["key"][0, t0].norm()
            inp["q"][1] = 0                                    # row 1: all energies 0: uniform
    row_len = torch.clamp(lens.repeat_interleave(N), 0, T)
    pad = torch.arange(T)[None] >= row_len[:, None]
    inp["key"][pad] = float("nan")
    inp["value"][pad] = float("nan")
    inp["pad"] = pad
    return inp


def _dev(t):
    return t.to(DEV).contiguous()


def _nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def run_case(pkg, name, inp, c0):
    """Forward, the non-accumulating backward (location kernels) and the accumulating backward of one case straight
    through the C ABI; -> dict of host tensors."""
    L, lib = pkg.lib, pkg.load_library()
    fam, _, T, D, E, K, R, temp, _, N, flags = CASES[name]
    rows, B = inp["q"].shape[0], rows_of(lib, name)
    cs = lib.b200asr_locattn_cluster_size(T, E)
    d = {k: _dev(v) for k, v in inp.items() if k != "pad"}
    attn, ctx = _nan(rows, T), _nan(rows, E)
    if fam == "loc":
        L.check(lib.b200asr_locattn_fwd(L.ptr(d["q"]), L.ptr(d["key"]), L.ptr(d["value"]), L.ptr(d["prev"]),
                                        L.ptr(d["lens"]), L.ptr(d["w_conv"]), L.ptr(d["w_proj"]), L.ptr(d["w_e"]),
                                        L.ptr(d["b_e"]), temp, B, T, D, E, K, R, L.ptr(attn), L.ptr(ctx), L.stream()),
                "locattn_fwd")
    else:
        L.check(lib.b200asr_dotattn_fwd(L.ptr(d["q"]), L.ptr(d["key"]), L.ptr(d["value"]), L.ptr(d["lens"]), N, temp,
                                        rows, T, D, E, L.ptr(attn), L.ptr(ctx), L.stream()), "dotattn_fwd")
    out = dict(attn=attn, ctx=ctx)
    if "fwd_only" not in flags:
        P = lib.b200asr_locattn_wpart_floats(D, K, R) if fam == "loc" else 0
        dkey_acc, wpart_acc = _dev(c0["dkey"]), (_dev(c0["wpart"]) if fam == "loc" else None)
        dq_acc = _nan(rows, cs, D)
        if fam == "loc":
            dq, dkey, dvalue, dprev, wpart = _nan(B, cs, D), _nan(B, T, D), _nan(B, T, E), _nan(B, T), _nan(B * cs, P)
            L.check(lib.b200asr_locattn_bwd(L.ptr(d["q"]), L.ptr(d["key"]), L.ptr(d["value"]), L.ptr(d["prev"]),
                                            L.ptr(d["lens"]), L.ptr(d["w_conv"]), L.ptr(d["w_proj"]), L.ptr(d["w_e"]),
                                            temp, L.ptr(attn), L.ptr(d["dctx"]), L.ptr(d["dattn"]), B, T, D, E, K, R,
                                            L.ptr(dq), L.ptr(dkey), L.ptr(dvalue), L.ptr(dprev), L.ptr(wpart),
                                            L.stream()), "locattn_bwd")
            dprev_acc = _nan(B, T)
            L.check(lib.b200asr_locattn_bwd_acc(L.ptr(d["q"]), L.ptr(d["key"]), L.ptr(d["value"]), L.ptr(d["prev"]),
                                                L.ptr(d["lens"]), L.ptr(d["w_conv"]), L.ptr(d["w_proj"]),
                                                L.ptr(d["w_e"]), temp, L.ptr(attn), L.ptr(d["dctx"]),
                                                L.ptr(d["dattn"]), B, T, D, E, K, R, L.ptr(dq_acc), L.ptr(dkey_acc),
                                                L.ptr(dprev_acc), L.ptr(wpart_acc), L.stream()), "locattn_bwd_acc")
            out.update(dq=dq, dkey=dkey, dvalue=dvalue, dprev=dprev, wpart=wpart, dprev_acc=dprev_acc,
                       wpart_acc=wpart_acc)
        else:
            L.check(lib.b200asr_dotattn_bwd_acc(L.ptr(d["q"]), L.ptr(d["key"]), L.ptr(d["value"]), L.ptr(d["lens"]),
                                                N, temp, L.ptr(attn), L.ptr(d["dctx"]), L.ptr(d["dattn"]), rows, T, D,
                                                E, L.ptr(dq_acc), L.ptr(dkey_acc), L.stream()), "dotattn_bwd_acc")
        out.update(dq_acc=dq_acc, dkey_acc=dkey_acc)
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in out.items()}


def _np(t):
    return t.double().numpy()


def check(tag, got, ref, bound):
    r = ar.worst_ratio(got, ref, bound)
    key = tag.split("/", 1)[1]                       # kernel/output, the worst over every case
    RATIOS[key] = max(RATIOS.get(key, 0.0), r)
    assert r <= 1.0, (tag, r)
    return r


def _loc_weights(inp):
    return inp["w_conv"].numpy(), inp["w_proj"].numpy(), inp["w_e"].numpy(), inp["b_e"].numpy()


def check_case(lib, name, inp, c0, out):
    fam, _, T, D, E, K, R, temp, _, N, flags = CASES[name]
    B, cs = rows_of(lib, name), lib.b200asr_locattn_cluster_size(T, E)
    n = lambda k: inp[k].double().numpy()
    args = dict(dctx=n("dctx"), dattn=n("dattn"), attn=_np(out["attn"])) if "fwd_only" not in flags else {}
    if fam == "loc":
        st = ar.loc_step(n("q"), n("key"), n("value"), n("prev"), inp["lens"].numpy(), *_loc_weights(inp), temp, **args)
    else:
        st = ar.dot_step(n("q"), n("key"), n("value"), inp["lens"].numpy(), N, temp, **args)
    valid = st.valid
    check("%s/%s_fwd/attn" % (name, fam), _np(out["attn"]), st.attn, np.where(valid, st.attn_b + TINY, 0.0))
    check("%s/%s_fwd/ctx" % (name, fam), _np(out["ctx"]), st.ctx, st.ctx_b)
    if "fwd_only" in flags:
        return
    pad = ~valid
    v3 = valid[:, :, None]
    c0k = c0["dkey"].double().numpy()
    got = _np(out["dkey_acc"])
    assert np.array_equal(out["dkey_acc"].view(torch.int32).numpy()[pad], c0["dkey"].view(torch.int32).numpy()[pad])
    check("%s/%s_bwd_acc/dkey" % (name, fam), got, np.where(v3, c0k + st.dkey, c0k),
          np.where(v3, st.dkey_b + 2 * ar.U * (np.abs(c0k) + st.dkey_abs), 0.0))
    check("%s/%s_bwd_acc/dq" % (name, fam), _np(out["dq_acc"]).sum(1), st.dq, st.dq_b)
    if fam != "loc":
        return
    check("%s/loc_bwd/dkey" % name, _np(out["dkey"]), st.dkey, st.dkey_b)
    check("%s/loc_bwd/dq" % name, _np(out["dq"]).sum(1), st.dq, st.dq_b)
    check("%s/loc_bwd/dvalue" % name, _np(out["dvalue"]), st.dvalue, st.dvalue_b)
    for k in ("dprev", "dprev_acc"):
        check("%s/loc_%s/dprev" % (name, "bwd" if k == "dprev" else "bwd_acc"), _np(out[k]), st.dprev, st.dprev_b)
    P, KW = lib.b200asr_locattn_wpart_floats(D, K, R), K * (2 * R + 1)
    pieces = [("dwp", 0, D * K), ("dwc", D * K, KW), ("dwe", D * K + KW, D), ("dbe", D * K + KW + D, 1)]
    for which in ("wpart", "wpart_acc"):
        wp = _np(out[which]).reshape(B, cs, P).sum(1)                   # per row, summed over the CTAs in float64
        base = c0["wpart"].double().numpy().reshape(B, cs, P).sum(1) if which == "wpart_acc" else 0 * wp
        base_abs = np.abs(c0["wpart"].double().numpy()).reshape(B, cs, P).sum(1) if which == "wpart_acc" else 0 * wp
        for f, o, m in pieces:
            val = getattr(st, f).reshape(B, -1)
            bnd = getattr(st, f + "_b").reshape(B, -1)
            ab = getattr(st, f + "_abs").reshape(B, -1)
            tag = "%s/loc_%s/%s" % (name, "bwd" if which == "wpart" else "bwd_acc", f)
            check(tag, wp[:, o:o + m], base[:, o:o + m] + val,
                  bnd + (cs + 1) * ar.U * (base_abs[:, o:o + m] + ab))


def _c0(lib, name, inp, seed):
    fam, _, T, D, E, K, R = CASES[name][:7]
    rows, B = inp["q"].shape[0], rows_of(lib, name)
    g = torch.Generator().manual_seed(seed)
    c0 = dict(dkey=torch.randn(rows, T, D, generator=g))
    if fam == "loc":
        cs = lib.b200asr_locattn_cluster_size(T, E)
        c0["wpart"] = torch.randn(B * cs, lib.b200asr_locattn_wpart_floats(D, K, R), generator=g)
    return c0


def _bits_equal(a, b):
    return all(torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)) for k in a)


@pytest.fixture(scope="module", autouse=True)
def _write_ratios():
    yield
    path = os.environ.get("ATTN_RATIOS_JSON")
    if path:
        with open(path, "w") as f:
            json.dump(RATIOS, f, indent=1, sort_keys=True)


@pytest.mark.parametrize("name", list(CASES))
def test_case_matches_float64_per_element(pkg, name):
    lib = pkg.load_library()
    fam, _, T, D, E, K, R, temp, _, N, flags = CASES[name]
    cls = case_classes(lib, name)
    cs = lib.b200asr_locattn_cluster_size(T, E)
    assert cs == ar.cluster_size(T, E) and "%s CS=%d" % (fam, cs) in cls
    if "fwd_only" not in flags:
        assert E // cs <= 1024 and minb(lib, name) in (1, 2)
        if fam == "dot":
            assert lib.b200asr_dotattn_supported(T, D, E) == 1 and pkg.ops.dot_attention_supported(T, D, E)
    inp = make_inputs(lib, name, seed=len(name) * 7 + T)
    c0 = _c0(lib, name, inp, seed=T + D)
    out = run_case(pkg, name, inp, c0)
    check_case(lib, name, inp, c0, out)
    assert _bits_equal(out, run_case(pkg, name, inp, c0)), "two runs differ"


def test_backward_limits(pkg):
    """The longest memory each backward takes at the configs' shapes runs within the bound; one frame more is refused
    before any launch."""
    L, lib = pkg.lib, pkg.load_library()
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    D, E, K, R = CFG["D"], CFG["E"], CFG["K"], CFG["R"]
    for fam, T in (("loc", loc_bwd_longest_t(optin)), ("dot", DOT_MAX_T)):
        name = "%s_limit" % fam
        CASES[name] = (fam, 2, T, D, E, K if fam == "loc" else 0, R if fam == "loc" else 0, 0.5, [T, T // 3], 1, ())
        try:
            inp = make_inputs(lib, name, seed=T)
            c0 = _c0(lib, name, inp, seed=T + 1)
            check_case(lib, name, inp, c0, run_case(pkg, name, inp, c0))
            CASES[name] = CASES[name][:2] + (T + 1,) + CASES[name][3:]
            inp = make_inputs(lib, name, seed=T)
            c0 = _c0(lib, name, inp, seed=T + 1)
            n0 = L.launch_count()
            with pytest.raises(L.B200AsrError, match="shared memory|frames >"):   # dot: the forward refuses too
                run_case(pkg, name, inp, c0)
            torch.cuda.synchronize()
            assert L.launch_count() == n0 + (1 if fam == "loc" else 0)   # the location forward itself still runs
        finally:
            del CASES[name]


@pytest.mark.parametrize("name", list(DVALUE))
def test_attn_dvalue_matches_float64(pkg, name):
    L, lib = pkg.lib, pkg.load_library()
    B, Ls, T, E, acc = DVALUE[name]
    Ls = dvalue_l(Ls)
    g = torch.Generator().manual_seed(Ls + T)
    a = torch.rand(B, Ls, T, generator=g)
    a[:, :, T // 2:] *= (torch.rand(B, Ls, T - T // 2, generator=g) < 0.5)     # exact zeros, as past len
    dc = torch.randn(B, Ls, E, generator=g)
    c0 = torch.randn(B, T, E, generator=g)
    out = _dev(c0) if acc else _nan(B, T, E)
    a_d, dc_d = _dev(a), _dev(dc)
    L.check(lib.b200asr_attn_dvalue(L.ptr(a_d), L.ptr(dc_d), B, Ls, T, E, L.ptr(out), acc, L.stream()), "attn_dvalue")
    ref, bnd = ar.dvalue(a.double().numpy(), dc.double().numpy(), c0.double().numpy() if acc else None)
    check("%s/attn_dvalue/dvalue" % name, _np(out.cpu()), ref, bnd)
    n0 = L.launch_count()
    with pytest.raises(L.B200AsrError, match="do not fit"):
        L.check(lib.b200asr_attn_dvalue(L.ptr(a_d), L.ptr(dc_d), B, dvalue_l(None) + 1, T, E, L.ptr(out), acc,
                                        L.stream()), "attn_dvalue")
    assert L.launch_count() == n0


# ------------------------------------------------------------------------------------------- the decode loop
def _decode_loop(pkg, fam, inp, Lsteps, temp, N=1):
    """L steps through ops.attention_memory and the *_mem_step functions; every step's d(attn) (for the location
    kernels: the loss's plus the next step's d(prev)) and d(q) captured."""
    lens = inp["lens"].to(DEV)
    leaves = {k: inp[k].to(DEV).requires_grad_(True) for k in ("qs", "key", "value") + (
        ("w_conv", "w_proj", "w_e", "b_e") if fam == "loc" else ())}
    if fam == "loc":
        mem, mk, mv, mcw, mpw, mew, meb, tok = pkg.ops.attention_memory(
            leaves["key"], leaves["value"], leaves["w_conv"].unsqueeze(1), leaves["w_proj"], leaves["w_e"].unsqueeze(0),
            leaves["b_e"])
    else:
        mem, mk, mv, tok = pkg.ops.attention_memory(leaves["key"], leaves["value"])
    prev, tot, steps, dattn = inp["prev"].to(DEV) if fam == "loc" else None, 0, [], {}
    for l in range(Lsteps):
        if fam == "loc":
            c, a = pkg.ops.loc_attention_mem_step(mem, tok, leaves["qs"][l], mk, mv, prev, lens, mcw, mpw, mew, meb,
                                                  temp)
        else:
            c, a = pkg.ops.dot_attention_mem_step(mem, tok, leaves["qs"][l], mk, mv, lens, N, temp)
        a.register_hook(lambda gr, l=l: dattn.__setitem__(l, gr.detach().cpu()))
        steps.append((prev.detach().cpu() if fam == "loc" else None, a.detach().cpu(), c.detach().cpu()))
        tot = tot + (c * inp["gc"][l].to(DEV)).sum() + (a * inp["ga"][l].to(DEV)).sum()
        prev = a
    tot.backward()
    return leaves, steps, dattn


@pytest.mark.parametrize("fam", ["loc", "dot"])
def test_decode_loop_per_element(pkg, fam):
    """Each step's forward from the GPU's own previous alignment, each step's backward from the GPU's own saved
    attention and d(attn); d(key), d(value) and the weight gradients accumulated over the loop."""
    lib = pkg.load_library()
    if fam == "loc":
        B, T, N, Ls, temp = 4, 149, 1, 12, 0.5
        D, E, K, R = CFG["D"], CFG["E"], CFG["K"], CFG["R"]
        lens = torch.tensor([149, 100, 38, 1])
    else:
        B, T, N, Ls, temp, D, E = 3, 37, 2, 8, 0.7, 64, 128
        lens = torch.tensor([37, 20, 1])
    rows = B * N
    g = torch.Generator().manual_seed(17)
    mk = lambda *s, sc=1.0: torch.randn(*s, generator=g) * sc
    inp = dict(lens=lens, qs=mk(Ls, rows, D), key=mk(rows, T, D), value=mk(rows, T, E), gc=mk(Ls, rows, E),
               ga=mk(Ls, rows, T))
    if fam == "loc":
        inp.update(prev=torch.rand(B, T, generator=g) / T, w_conv=mk(K, 2 * R + 1, sc=0.3), w_proj=mk(D, K, sc=0.5),
                   w_e=mk(D, sc=0.3), b_e=mk(1))
    pad = torch.arange(T)[None] >= torch.clamp(lens.repeat_interleave(N), 0, T)[:, None]
    inp["key"][pad] = float("nan")
    inp["value"][pad] = float("nan")
    leaves, steps, dattn = _decode_loop(pkg, fam, inp, Ls, temp, N)
    n = lambda t: t.double().numpy()
    acc = {k: [] for k in ("dkey", "dwp", "dwc", "dwe", "dbe")}
    for l, (prev, a, c) in enumerate(steps):
        args = dict(dctx=n(inp["gc"][l]), dattn=n(dattn[l]), attn=n(a))
        if fam == "loc":
            st = ar.loc_step(n(inp["qs"][l]), n(inp["key"]), n(inp["value"]), n(prev), lens.numpy(),
                             *(n(inp[k]) for k in ("w_conv", "w_proj", "w_e", "b_e")), temp, **args)
        else:
            st = ar.dot_step(n(inp["qs"][l]), n(inp["key"]), n(inp["value"]), lens.numpy(), N, temp, **args)
        check("decode_%s/%s_fwd/attn" % (fam, fam), n(a), st.attn, np.where(st.valid, st.attn_b + TINY, 0.0))
        check("decode_%s/%s_fwd/ctx" % (fam, fam), n(c), st.ctx, st.ctx_b)
        cs = lib.b200asr_locattn_cluster_size(T, E)
        check("decode_%s/%s_bwd_acc/dq" % (fam, fam), n(leaves["qs"].grad[l].cpu()), st.dq,
              st.dq_b + (cs + 1) * ar.U * st.dq_abs)
        if fam == "loc" and l > 0:      # d(attn of step l-1) = the loss's + this step's d(prev)
            check("decode_loc/loc_bwd_acc/dprev", n(dattn[l - 1]), n(inp["ga"][l - 1]) + st.dprev,
                  st.dprev_b + 2 * ar.U * (np.abs(n(inp["ga"][l - 1])) + st.dprev_abs))
        for k in acc:
            if hasattr(st, k):
                acc[k].append((getattr(st, k), getattr(st, k + "_b"), getattr(st, k + "_abs")))
    v3 = (np.arange(T)[None] < np.clip(lens.repeat_interleave(N).numpy(), 0, T)[:, None])[:, :, None]
    val, bnd = ar.accumulate(0.0, *zip(*acc["dkey"]))
    check("decode_%s/%s_bwd_acc/dkey" % (fam, fam), n(leaves["key"].grad.cpu()), val, np.where(v3, bnd, 0.0))
    dv, dvb = ar.dvalue(np.stack([n(a) for _, a, _ in steps], 1), n(inp["gc"].transpose(0, 1)))
    check("decode_%s/attn_dvalue/dvalue" % fam, n(leaves["value"].grad.cpu()), np.where(v3, dv, 0.0),
          np.where(v3, dvb, 0.0))
    if fam == "loc":
        for k, leaf, shape in (("dwp", "w_proj", (D, K)), ("dwc", "w_conv", (K, 2 * R + 1)), ("dwe", "w_e", (D,)),
                               ("dbe", "b_e", (1,))):
            vals, bnds, abss = zip(*acc[k])
            val, bnd = ar.accumulate(0.0, [v.sum(0) for v in vals], [b.sum(0) for b in bnds], [a.sum(0) for a in abss])
            bnd = bnd + B * cs * ar.U * sum(a.sum(0) for a in abss)
            check("decode_loc/loc_bwd_acc/%s" % k, n(leaves[leaf].grad.cpu()).reshape(shape), val.reshape(shape),
                  bnd.reshape(shape))


# ------------------------------------------------------------------------------------------- len = 0
def _ref_nan_pattern(fam, inp, T, N, temp):
    """Float64 autograd of the reference's expressions (one step): which outputs and gradients are NaN."""
    from test_gpu_dot_attention import _dot_attention_torch
    from test_gpu_kernel_variants import _loc_attention_torch
    key = inp["key"].double().nan_to_num(0.0)
    value = inp["value"].double().nan_to_num(0.0)
    x = [t.requires_grad_(True) for t in (inp["qs"][0].double(), key, value)]
    if fam == "loc":
        w = [inp[k].double() for k in ("w_conv", "w_proj", "w_e", "b_e")]
        c, a = _loc_attention_torch(x[0], x[1], x[2], inp["prev"].double(), inp["lens"], w[0].unsqueeze(1), w[1],
                                    w[2].unsqueeze(0), w[3], temp)
    else:
        c, a = _dot_attention_torch(x[0], x[1], x[2], inp["lens"], N, temp)
    ((c * inp["gc"][0].double()).sum() + (a * inp["ga"][0].double()).sum()).backward()
    return [torch.isnan(t) for t in (c.detach(), a.detach(), x[0].grad, x[1].grad, x[2].grad)]


@pytest.mark.parametrize("fam", ["loc", "dot"])
def test_empty_utterance_gives_the_reference_nan(pkg, fam):
    """enc_len 0: the reference's softmax of an all -inf row is NaN, and so are its context and d(value); d(key) and
    d(q) stay 0 (masked_fill's backward).  The loss is NaN, so the fused optimizer skips the step."""
    B, T, N, D, E, K, R, temp = 2, 40, 1, 16, 64, 3, 4, 0.5
    g = torch.Generator().manual_seed(3)
    mk = lambda *s: torch.randn(*s, generator=g)
    inp = dict(lens=torch.tensor([T, 0]), qs=mk(1, B, D), key=mk(B, T, D), value=mk(B, T, E), gc=mk(1, B, E),
               ga=mk(1, B, T), prev=torch.rand(B, T, generator=g) / T, w_conv=mk(K, 2 * R + 1), w_proj=mk(D, K),
               w_e=mk(D), b_e=mk(1))
    inp["key"][1] = float("nan")
    inp["value"][1] = float("nan")
    leaves, steps, _ = _decode_loop(pkg, fam, inp, 1, temp)
    _, a, c = steps[0]
    got = [torch.isnan(t) for t in (c, a, leaves["qs"].grad[0].cpu(), leaves["key"].grad.cpu(),
                                    leaves["value"].grad.cpu())]
    for name, x, y in zip(("ctx", "attn", "d(q)", "d(key)", "d(value)"), got, _ref_nan_pattern(fam, inp, T, N, temp)):
        assert torch.equal(x, y), name
    assert bool(got[0][1].all()) and not bool(got[0][0].any()) and bool(got[4][1].all())
    assert float(leaves["key"].grad[1].abs().max()) == 0
    loss = (c * inp["gc"][0]).sum()
    assert math.isnan(loss.item())


def test_empty_utterance_under_graph_replay(pkg):
    """A location step (forward, accumulating backward, d(value)) captured on full lengths and replayed with one
    length set to 0: that row's context and d(value) become NaN, the other row is unchanged, and a replay on full
    lengths is finite again."""
    L, lib = pkg.lib, pkg.load_library()
    B, T, D, E, K, R, temp = 2, 40, 16, 64, 3, 4, 0.5
    g = torch.Generator().manual_seed(4)
    mk = lambda *s: torch.randn(*s, generator=g).to(DEV)
    q, key, value, dctx = mk(B, D), mk(B, T, D), mk(B, T, E), mk(B, E)
    prev = (torch.rand(B, T, generator=g) / T).to(DEV)
    wc, wp, we, be = mk(K, 2 * R + 1), mk(D, K), mk(D), mk(1)
    lens = torch.full((B,), T, dtype=torch.int64, device=DEV)
    cs = lib.b200asr_locattn_cluster_size(T, E)
    attn, ctx, dq, dprev = (torch.empty(B, T, device=DEV), torch.empty(B, E, device=DEV),
                            torch.empty(B, cs, D, device=DEV), torch.empty(B, T, device=DEV))
    dkey, dvalue = torch.zeros(B, T, D, device=DEV), torch.zeros(B, T, E, device=DEV)
    wpart = torch.zeros(B * cs, lib.b200asr_locattn_wpart_floats(D, K, R), device=DEV)

    def step():
        dkey.zero_()
        wpart.zero_()
        L.check(lib.b200asr_locattn_fwd(L.ptr(q), L.ptr(key), L.ptr(value), L.ptr(prev), L.ptr(lens), L.ptr(wc),
                                        L.ptr(wp), L.ptr(we), L.ptr(be), temp, B, T, D, E, K, R, L.ptr(attn),
                                        L.ptr(ctx), L.stream()))
        L.check(lib.b200asr_locattn_bwd_acc(L.ptr(q), L.ptr(key), L.ptr(value), L.ptr(prev), L.ptr(lens), L.ptr(wc),
                                            L.ptr(wp), L.ptr(we), temp, L.ptr(attn), L.ptr(dctx), None, B, T, D, E, K,
                                            R, L.ptr(dq), L.ptr(dkey), L.ptr(dprev), L.ptr(wpart), L.stream()))
        L.check(lib.b200asr_attn_dvalue(L.ptr(attn), L.ptr(dctx), B, 1, T, E, L.ptr(dvalue), 0, L.stream()))

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    eager = [t.clone() for t in (ctx, dvalue, dkey)]
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    lens.fill_(T)
    lens[1] = 0
    graph.replay()
    torch.cuda.synchronize()
    assert bool(torch.isnan(ctx[1]).all()) and bool(torch.isnan(dvalue[1]).all())
    assert float(dkey[1].abs().max()) == 0
    assert torch.equal(ctx[0], eager[0][0]) and torch.equal(dvalue[0], eager[1][0]) and torch.equal(dkey[0], eager[2][0])
    lens.fill_(T)
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip((ctx, dvalue, dkey), eager))
