"""The f16x3 GEMM (scaled fp16 hi/lo images, csrc/gemm.cu) against float64: the four BiLSTM layer contractions at
cfg-B shapes, tails / accumulate / bias / ldc / gate permutation, the shifted h_prev image, rows and utterance blocks
far apart in magnitude, NaN / Inf propagation and run-to-run bit equality."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
H, B, T = 512, 64, 1198          # cfg B: hidden size, utterances, frames of layer 0 (B * T = 76672 rows)


def _err(out, ref):
    """max |out - ref| / max |ref| (float64)"""
    return float((out.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-300))


def _sgemm(a, b):
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        return a @ b
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


def _perm_rows(ref):
    M = ref.shape[0]
    idx = torch.arange(M, device=ref.device)
    out = torch.empty_like(ref)
    out[(idx % 4) * (M // 4) + idx // 4] = ref
    return out


def _check(out, ref, sgemm):
    e, es = _err(out, ref), _err(sgemm, ref)
    assert e < 3e-6 and e <= 20 * max(es, 2.0 ** -24), (e, es)


@pytest.mark.parametrize("M,N,K", [(B * T, 4 * H, 1024),     # layer-1 input projection
                                   (B * T, 1024, 4 * H)])    # layer-1 input gradient dX = dG . W
def test_tn_forms_vs_fp64(pkg, M, N, K):
    ops = pkg.ops
    torch.manual_seed(M + N + K)
    a = torch.randn(M, K, device=DEV)
    w = torch.randn(N, K, device=DEV) * 0.05
    bias = torch.randn(N, device=DEV)
    ai, wi = ops.f16_split(a, M, K), ops.f16_split(w, N, K)
    out = ops.gemm_f16x3(ai, wi, bias=bias)
    assert torch.equal(out, ops.gemm_f16x3(ai, wi, bias=bias))            # two runs bit-identical
    ref = a.double() @ w.double().t() + bias.double()
    _check(out, ref, _sgemm(a, w.t()) + bias)


@pytest.mark.parametrize("N", [1024, 120])
def test_weight_gradient_vs_fp64(pkg, N):
    """dW_ih = dG^T . X over all 76672 rows of a cfg-B batch, gate permutation in the epilogue."""
    ops = pkg.ops
    torch.manual_seed(N)
    g = torch.randn(B * T, 4 * H, device=DEV)
    x = torch.randn(B * T, N, device=DEV)
    gt, xt = ops.f16_split_t(g, 4 * H, B * T), ops.f16_split_t(x, N, B * T)
    out = ops.gemm_f16x3(gt, xt, permute_rows=True, name="gemm_f16_nt")
    assert torch.equal(out, ops.gemm_f16x3(gt, xt, permute_rows=True, name="gemm_f16_nt"))
    ref = _perm_rows(g.double().t() @ x.double())
    _check(out, ref, _perm_rows(_sgemm(g.t(), x)))


def _hprev(h, d, Tn):
    """h_prev of direction d from the layer output h[b, t, d*H:(d+1)*H] (zero at the direction's first step)"""
    hd = h[:, :, d * H:(d + 1) * H].double()
    hp = torch.zeros_like(hd)
    if d == 0:
        hp[:, 1:] = hd[:, :-1]
    else:
        hp[:, :-1] = hd[:, 1:]
    return hp.reshape(-1, H)


@pytest.mark.parametrize("Bn,Tn", [(B, T), (3, 5)])
def test_weight_gradient_shifted_hprev(pkg, Bn, Tn):
    """dW_hh = dG^T . h_prev with h_prev's image written shifted by one step per utterance, both directions."""
    ops = pkg.ops
    torch.manual_seed(Tn)
    h = torch.randn(Bn, Tn, 2 * H, device=DEV)
    for d in range(2):
        g = torch.randn(Bn * Tn, 4 * H, device=DEV)
        ht = ops.f16_split_t(h[:, :, d * H:(d + 1) * H], H, Tn, batches=Bn, ld=2 * H, bstride=Tn * 2 * H,
                             shift=(-1 if d == 0 else 1))
        out = ops.gemm_f16x3(ops.f16_split_t(g, 4 * H, Bn * Tn), ht, permute_rows=True)
        hp = _hprev(h, d, Tn)
        ref = _perm_rows(g.double().t() @ hp)
        _check(out, ref, _perm_rows(_sgemm(g.t(), hp.float())))


@pytest.mark.parametrize("M,N,K,acc,pad", [(77, 31, 120, False, 0), (77, 36, 132, True, 5), (64, 1024, 2048, True, 3),
                                           (300, 130, 4, False, 2)])
def test_tails_accumulate_bias_ldc(pkg, M, N, K, acc, pad):
    """M / N / K not multiples of 128 or 16, accumulate into C, bias, ldc > N, split-K (M = 64)."""
    ops = pkg.ops
    torch.manual_seed(M * N + K)
    a = torch.randn(M, K, device=DEV)
    w = torch.randn(N, K, device=DEV)
    bias = torch.randn(N, device=DEV)
    base = torch.randn(M, N + pad, device=DEV)
    out = base.clone()
    ops.gemm_f16x3(ops.f16_split(a, M, K), ops.f16_split(w, N, K), bias=bias, out=out[:, :N], accumulate=acc)
    ref = a.double() @ w.double().t() + bias.double() + (base[:, :N].double() if acc else 0)
    assert _err(out[:, :N], ref) < 3e-6
    assert torch.equal(out[:, N:], base[:, N:])                          # columns beyond N untouched


def test_nt_tails_and_permutation(pkg):
    ops = pkg.ops
    torch.manual_seed(7)
    R, M, N = 1000, 132, 36
    a, b = torch.randn(R, M, device=DEV), torch.randn(R, N, device=DEV)
    out = ops.gemm_f16x3(ops.f16_split_t(a, M, R), ops.f16_split_t(b, N, R), permute_rows=True)
    assert _err(out, _perm_rows(a.double().t() @ b.double())) < 3e-6


def test_dynamic_range_rows(pkg):
    """dG rows at 2^-40 ... 2^+20 and zero rows: every row of dX = dG . W keeps its own fp32-class accuracy."""
    ops = pkg.ops
    torch.manual_seed(11)
    M, N, K = 4096, 1024, 2048
    g = torch.randn(M, K, device=DEV)
    e = torch.randint(-40, 21, (M, 1), device=DEV).float()
    g = g * torch.exp2(e)
    g[::97] = 0
    w = torch.randn(N, K, device=DEV) * 0.05
    out = ops.gemm_f16x3(ops.f16_split(g, M, K), ops.f16_split(w, N, K))
    ref = g.double() @ w.double().t()
    zero = g.abs().amax(1) == 0
    assert torch.all(out[zero] == 0)
    row_err = (out.double() - ref).abs().amax(1) / ref.abs().amax(1).clamp_min(1e-300)
    assert float(row_err[~zero].max()) < 3e-6


def test_dynamic_range_utterance_blocks(pkg):
    """Utterance blocks of dG at 2^-40 ... 2^+20 (blocks of T rows, not aligned to the 128-row scale chunks) with X
    scaled inversely, so that every block matters in dW = dG^T . X; zero utterances."""
    ops = pkg.ops
    torch.manual_seed(12)
    Bn, Tn, M, N = 40, 301, 2048, 512
    ex = torch.linspace(-40, 20, Bn, device=DEV).round().view(Bn, 1, 1)
    g = torch.randn(Bn, Tn, M, device=DEV) * torch.exp2(ex)
    x = torch.randn(Bn, Tn, N, device=DEV) * torch.exp2(-ex - 10)
    g[5] = 0
    g2, x2 = g.view(-1, M), x.view(-1, N)
    out = ops.gemm_f16x3(ops.f16_split_t(g2, M, Bn * Tn), ops.f16_split_t(x2, N, Bn * Tn))
    ref = g2.double().t() @ x2.double()
    _check(out, ref, _sgemm(g2.t(), x2))


def test_nan_inf_poison_the_outputs_fp32_would(pkg):
    """A NaN / Inf in an operand makes exactly the outputs non-finite that an fp32 GEMM makes non-finite."""
    ops = pkg.ops
    torch.manual_seed(13)
    M, N, K = 300, 260, 520
    a, w = torch.randn(M, K, device=DEV), torch.randn(N, K, device=DEV)
    a[3, 7] = float("nan")
    a[200, 300] = float("inf")
    a[201, 0] = float("-inf")
    a[201, 1] = 1e30                     # finite, far beyond fp16, in the chunk of an Inf
    w[17, 130] = float("nan")
    w[250, 519] = float("inf")
    out = ops.gemm_f16x3(ops.f16_split(a, M, K), ops.f16_split(w, N, K))
    ref = _sgemm(a, w.t())
    assert torch.equal(torch.isfinite(out), torch.isfinite(ref))
    fin = torch.isfinite(ref)
    exact = a.double().nan_to_num(0, 0, 0) @ w.double().nan_to_num(0, 0, 0).t()
    assert _err(out[fin], exact[fin]) < 3e-6
    # the weight-gradient form: a NaN in dG^T's image poisons its gate row, an Inf in X its column
    g, x = torch.randn(1000, 64, device=DEV), torch.randn(1000, 36, device=DEV)
    g[500, 9] = float("nan")
    x[20, 4] = float("inf")
    out = ops.gemm_f16x3(ops.f16_split_t(g, 64, 1000), ops.f16_split_t(x, 36, 1000))
    assert torch.equal(torch.isfinite(out), torch.isfinite(_sgemm(g.t(), x)))
