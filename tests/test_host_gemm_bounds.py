"""CPU checks for tests/test_gpu_gemm_parity.py: the split-K plan the dispatcher reports matches a restatement of the
rule, the GPU file's cases reach the plans they name, its exact generators satisfy the grid condition, and its
per-element bound has teeth.

The 3xTF32 arithmetic is emulated in numpy: a_hi = trunc_tf32(a), a_lo = a - a_hi read truncated again by the tensor
core, products a_hi b_hi + a_lo b_hi + a_hi b_lo per 8 k, each MMA instruction adding its exact product sum to the
running fp32 accumulator with truncation (the accumulation model of the bound), chunks of 4 K blocks folded with IEEE
adds, split-K partial tiles summed in slice order, then the bias and C0.  The correct emulation must stay at or below
half the bound on the GPU file's input generators; each defect a kernel could plausibly have must exceed it 4x.
"""
import numpy as np
import pytest
import torch

import test_gpu_gemm_parity as P

U = 2.0 ** -24


# ------------------------------------------------------------------------------------------------ plan table
def _pick(M, N, KB, sms):
    tiles = -(-M // 128) * -(-N // 128)
    s = max(1, min(sms // tiles, KB // 8, 32))
    rule = "sm_fill" if s > 1 else "one"
    eff = lambda q: tiles * q / (-(-tiles * q // sms) * sms)          # noqa: E731
    if 2 * tiles <= sms and eff(s) < 0.93:
        cap = max(1, min(32, (160 << 20) // max(M * N * 4, 1)))
        q = s + 1
        while q <= cap and KB // q >= 64:
            if eff(q) >= 0.97:
                return q, "efficiency"
            q += 1
    return s, rule


def plan_restated(form, M, N, K, batches, ws, sms=132, chunk=4):
    """The split rule of csrc/gemm.cu in Python."""
    if form == "f16x3":
        KB, unit, rule_kb, ch, bk = -(-K // 128) * 2, 2, -(-K // 128) * 4, 2, 64
    else:
        KB, unit, ch, bk = -(-K // 32) * (batches if form == "nt" else 1), 1, chunk, 32
        rule_kb = KB
    req, rule = _pick(M, N, rule_kb, sms)
    n = req
    if n > 1 and ws < n * M * N * 4:
        n, rule = 1, "workspace"
    kps = -(-(KB // unit) // n) * unit
    n = -(-KB // kps)
    last = KB - (n - 1) * kps
    return dict(rule=rule, requested=req, nsplit=n, kb_per_split=kps, kb_last=last, chunk=ch,
                last_chunk_first=(min(KB, kps) - 1) % ch + 1, last_chunk_last=(last - 1) % ch + 1, KB=KB, bk=bk)


def _sweep():
    rng = np.random.default_rng(0)
    for _ in range(400):
        form = ("tn", "tn_pre", "nn", "nt", "f16x3")[rng.integers(5)]
        M, N = int(rng.integers(1, 6000)), int(rng.integers(1, 3000))
        if rng.random() < 0.5:
            M = int(rng.integers(1, 300))
        K = int(rng.integers(1, 90000))
        bt = int(rng.integers(1, 70)) if form == "nt" else 1
        if form == "nt":
            K = max(1, K // bt)
        ws = (0, 16, 1 << 20, None)[rng.integers(4)]
        yield form, M, N, K, bt, ws
    for form, M, N, K, bt, ws in P.CANDIDATES:
        yield form, M, N, K, bt, ws


def test_plan_query_matches_the_rule(pkg):
    lib = pkg.load_library()
    if lib.b200asr_device_sm_count() != 132:
        pytest.skip("the restatement is checked at 132 SMs")
    rules = set()
    for form, M, N, K, bt, ws in _sweep():
        wsb = lib.b200asr_gemm3x_workspace_bytes(M, N) if ws is None else ws
        got = P.gemm_plan(lib, form, M, N, K, bt, wsb)
        assert got == plan_restated(form, M, N, K, bt, wsb), (form, M, N, K, bt, wsb)
        rules.add(got["rule"])
    assert rules == set(P.RULES)


def test_plan_query_rejects_bad_arguments(pkg):
    import ctypes
    lib = pkg.load_library()
    d = (ctypes.c_int * 10)()
    assert lib.b200asr_debug_gemm_plan(5, 64, 64, 64, 1, 0, d) == -1
    assert lib.b200asr_debug_gemm_plan(0, 64, 64, 64, 2, 0, d) == -1          # batches only for nt
    assert lib.b200asr_debug_gemm_plan(3, 64, 64, 0, 2, 0, d) == -1


def test_gpu_cases_reach_the_plans_they_name(pkg):
    """At 132 SMs: every plan class has a candidate, and the production cases reach the rule they name."""
    lib = pkg.load_library()
    if lib.b200asr_device_sm_count() != 132:
        pytest.skip("the table is stated for 132 SMs")
    assert set(P.CLASSES) <= set(P.class_cases(lib))
    for name, form, M, N, K, opt, rule in P.PRODUCTION:
        assert P.production_plan(lib, form, M, N, K, opt)["rule"] == rule, name


# ------------------------------------------------------------------------------------------------ exact generators
@pytest.mark.parametrize("kind", ["int", "res_a", "res_b"])
@pytest.mark.parametrize("K", [132, 1000, 8196, 76672])
def test_exact_generators_satisfy_the_grid_condition(kind, K):
    """The worst case of each generator pair (not only a sample) keeps 2^g (S + |bias| + |C0|) below 2^24, and a
    sample of the residual kinds is not exact without the lo products."""
    ka, kb = P.EXACT_KINDS[kind]
    lim = {"int": 7, "int2": 2, "res": 2 - 2.0 ** -12}
    nnz = min(K, P.RES_NNZ) if "res" in (ka, kb) else K
    g = 0 if kind == "int" else 12
    extra = 64 + (1 << 20) if kind == "int" else 64 + 64
    assert 2.0 ** g * (nnz * lim[ka] * lim[kb] + extra) < 2.0 ** 24
    gen = torch.Generator().manual_seed(K)
    a = P.grid_operand(ka, 6, K, gen, device="cpu").double()
    b = P.grid_operand(kb, 5, K, gen, device="cpu", phase=5).double()
    r = a if ka == "res" else b
    assert int((r != 0).sum(1).max()) <= nnz               # nonzero products per output
    assert float(a.abs().max()) <= lim[ka] and float(b.abs().max()) <= lim[kb]
    assert torch.equal(a * 2.0 ** g, (a * 2.0 ** g).round()) and torch.equal(b * 2.0 ** g, (b * 2.0 ** g).round())
    if kind != "int":
        hi = torch.from_numpy(_tf32(a.numpy())), torch.from_numpy(_tf32(b.numpy()))
        assert not torch.equal(hi[0] @ hi[1].t(), a @ b.t())
        lo = r.numpy() - _tf32(r.numpy())                # the residual is TF32-exact: the tensor core's truncation
                                                         # of lo loses nothing
        assert np.array_equal(_tf32(lo), lo)


# ------------------------------------------------------------------------------------------------ emulated 3xTF32
def _tf32(x):
    return (np.asarray(x, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32).astype(np.float64)


def _trunc32(x):
    """float64 -> the fp32 value next to it towards zero"""
    f = x.astype(np.float32)
    over = np.abs(f.astype(np.float64)) > np.abs(x)
    f[over] = np.nextafter(f[over], np.float32(0))
    return f.astype(np.float64)


def emulate(a, b, bias, c0, *, nsplit=1, ch=4, drop_alo=False, drop_blo=False, drop_block=False, bias_per_slice=False,
            stale_blo=False, no_chunks=False):
    """C = a[M, K] . b[K, N] + bias + c0 as the 3xTF32 kernel computes it (a, b fp32 values as float64)."""
    M, K = a.shape
    KB = -(-K // 32)
    Kp = KB * 32
    a = np.pad(a, ((0, 0), (0, Kp - K)))
    b = np.pad(b, ((0, Kp - K), (0, 0)))
    ah, bh = _tf32(a), _tf32(b)
    al, bl = _tf32(a - ah), _tf32(b - bh)
    if drop_alo:
        al = al * 0
    if drop_blo:
        bl = bl * 0
    if stale_blo:                                      # B's residual of the previous K block
        bl = np.concatenate([bl[:32], bl[:-32]])
    kps = -(-KB // nsplit)
    out = np.zeros((M, b.shape[1]))
    for s in range(-(-KB // kps)):
        blocks = list(range(s * kps, min(KB, (s + 1) * kps)))
        if drop_block and s == 1:
            blocks = blocks[1:]
        acc = np.zeros_like(out)
        chunk = len(blocks) if no_chunks else ch
        for c0_ in range(0, len(blocks), chunk):
            d = np.zeros_like(out)
            for kb in blocks[c0_:c0_ + chunk]:
                for k8 in range(kb * 32, kb * 32 + 32, 8):
                    sl = slice(k8, k8 + 8)
                    d = _trunc32(d + ah[:, sl] @ bh[sl] + al[:, sl] @ bh[sl] + ah[:, sl] @ bl[sl])
            acc = (acc.astype(np.float32) + d.astype(np.float32)).astype(np.float64)
        if bias_per_slice:
            acc = (acc.astype(np.float32) + bias.astype(np.float32)).astype(np.float64)
        out = (out.astype(np.float32) + acc.astype(np.float32)).astype(np.float64)
    out = (out.astype(np.float32) + bias.astype(np.float32)).astype(np.float64)
    return (out.astype(np.float32) + c0.astype(np.float32)).astype(np.float64)


def _bound(a, b, bias, c0, nsplit, ch=4):
    S = np.abs(a) @ np.abs(b)
    KB = -(-a.shape[1] // 32)
    chunks = -(-KB // ch) + nsplit
    floor = 2.0 ** -135 * (np.abs(a).sum(1, keepdims=True) + np.abs(b).sum(0, keepdims=True))
    return ((3 * 2.0 ** -20 + 2 * 2.0 ** -23 * 12 * ch) * S + (chunks + nsplit + 2) * U * (S + np.abs(bias) + np.abs(c0))
            + floor)


def _operands(kind, M, N, K, seed):
    g = torch.Generator().manual_seed(seed)
    a = P.bound_operand(kind, M, K, g, "a", device="cpu").double().numpy()
    b = P.bound_operand(kind, N, K, g, "b", device="cpu").double().numpy().T
    rng = np.random.default_rng(seed)
    return a, b, rng.standard_normal(N).astype(np.float32).astype(np.float64), \
        rng.standard_normal((M, N)).astype(np.float32).astype(np.float64)


MUTATIONS = {"A_lo.B dropped": dict(drop_alo=True), "A_hi.B_lo dropped": dict(drop_blo=True),
             "K block dropped at a slice boundary": dict(drop_block=True), "bias added per slice": dict(bias_per_slice=True),
             "B residual from a stale tile": dict(stale_blo=True)}


def test_bound_accepts_the_kernel_arithmetic_and_rejects_defects():
    M, N, K, nsplit = 6, 5, 300, 3
    worst = {}
    for kind in ("pos", "cancel", "range", "zero_subnormal"):
        a, b, bias, c0 = _operands(kind, M, N, K, len(kind))
        exact = a @ b + bias + c0
        bnd = _bound(a, b, bias, c0, nsplit)
        r = float((np.abs(emulate(a, b, bias, c0, nsplit=nsplit) - exact) / bnd).max())
        assert r <= 0.5, (kind, r)
        for name, kw in MUTATIONS.items():
            e = np.abs(emulate(a, b, bias, c0, nsplit=nsplit, **kw) - exact) / bnd
            worst[name] = max(worst.get(name, 0.0), float(np.nanmax(e)))
    print(worst)
    for name, r in worst.items():
        assert r >= 4, (name, r)


def test_bound_rejects_a_shift_off_by_one():
    """nt with b_shift = -1 read as 0: the rows of B meet the wrong rows of A."""
    a, b, bias, c0 = _operands("pos", 6, 5, 640, 3)
    bs = np.zeros_like(b)
    bs[1:] = b[:-1]                                    # B[t - 1]
    exact = a @ bs + bias + c0
    r = float((np.abs(emulate(a, b, bias, c0) - exact) / _bound(a, bs, bias, c0, 1)).max())
    assert r >= 4, r


def test_bound_rejects_one_chain_over_all_of_k():
    """Without the chunk folds the tensor core's truncating accumulate runs over the whole cfg-B depth (76672 k):
    all-positive operands make that coherent."""
    a, b, bias, c0 = _operands("pos", 2, 2, 76672, 9)
    exact = a @ b + bias + c0
    bnd = _bound(a, b, bias, c0, 1)
    r_ok = float((np.abs(emulate(a, b, bias, c0) - exact) / bnd).max())
    r_bad = float((np.abs(emulate(a, b, bias, c0, no_chunks=True) - exact) / bnd).max())
    print(r_ok, r_bad)
    assert r_ok <= 0.5 and r_bad >= 4, (r_ok, r_bad)
