"""The 3xTF32 GEMM main loop (A fragments split in registers, MMAs of consecutive K blocks in flight) at the shapes of
the cfg-B train step: the input gradient through the tn form on a transposed weight against the nn form and fp64,
the weight gradients at the full contraction depth, and every accumulation chunk length."""
import os
import subprocess
import sys

import pytest
import torch

from conftest import scaled_err

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _tn_vs_nn(ops, M, N, K, acc):
    """dX[M,N] (+)= dG[M,K] . W[K,N] as gemm_tn(dG, W^T, w_lo=residual(W^T)) and, where the nn form takes the row
    pitch (N % 4 == 0), as gemm_nn(dG, W)."""
    torch.manual_seed(M + N + K)
    g = torch.randn(M, K, device=DEV)
    w = torch.randn(K, N, device=DEV) * 0.05
    c0 = torch.randn(M, N, device=DEV)
    wt = w.t().contiguous()
    out_tn, out_nn = c0.clone(), None
    ops.gemm_tn(g, wt, out=out_tn, accumulate=acc, w_lo=ops.tf32_residual(wt))
    if N % 4 == 0:
        out_nn = c0.clone()
        ops.gemm_nn(g, w, out=out_nn, accumulate=acc)
    ref = g.double() @ w.double() + (c0.double() if acc else 0)
    return out_tn, out_nn, ref


@pytest.mark.parametrize("M,N,K,acc", [
    (19136, 2048, 2048, True),     # cfg-B layer 3, second direction accumulates
    (77, 31, 120, False),          # M / N / K tails (N % 4 != 0: the nn form does not take this pitch)
    (77, 36, 120, True),           # the same tails, comparable with the nn form
    (64, 1024, 2048, True),        # skinny: split-K slices
])
def test_input_gradient_tn_on_transposed_weight(pkg, M, N, K, acc):
    out_tn, out_nn, ref = _tn_vs_nn(pkg.ops, M, N, K, acc)
    for out in (out_tn, out_nn):
        if out is not None:
            assert scaled_err(out.cpu().numpy(), ref.cpu().numpy()) < 3e-6
    if out_nn is None:
        return
    # same hi / lo values and the same MMA sequence: the tn form reads B's raw fp32 tile as its hi operand, the nn form
    # an explicitly truncated one, so this holds because the tensor core truncates a raw fp32 tf32 operand
    assert torch.equal(out_tn, out_nn)


def _nt_check(ops, M, N, T, batches, shift, perm, cols=64):
    torch.manual_seed(M + T)
    a = torch.randn(batches, T, M, device=DEV)
    b = torch.randn(batches, T, N, device=DEV)
    args = dict(batches=batches, a_bstride=T * M, b_bstride=T * N, b_shift=shift, permute_rows=perm)
    out = ops.gemm_nt(a, b, M, N, T, **args)
    assert torch.equal(out, ops.gemm_nt(a, b, M, N, T, **args))            # repeated runs are bit-equal
    bs = torch.zeros(batches, T, cols, device=DEV, dtype=torch.float64)
    if shift == 0:
        bs[:] = b[:, :, :cols].double()
    elif shift < 0:
        bs[:, 1:] = b[:, :-1, :cols].double()
    else:
        bs[:, :-1] = b[:, 1:, :cols].double()
    ref = torch.einsum("btm,btn->mn", a.double(), bs)
    if perm:
        idx = torch.arange(M, device=DEV)
        r2 = torch.empty_like(ref)
        r2[(idx % 4) * (M // 4) + idx // 4] = ref
        ref = r2
    assert scaled_err(out[:, :cols].cpu().numpy(), ref.cpu().numpy()) < 3e-6


@pytest.mark.parametrize("N", [1024, 120])
def test_weight_gradient_full_contraction_depth(pkg, N):
    """dW_ih = dG^T . X over all 76672 rows of a cfg-B batch (the layer-1 and layer-0 input widths)."""
    _nt_check(pkg.ops, 2048, N, 76672, 1, 0, True)


@pytest.mark.parametrize("shift", [-1, 1])
def test_recurrent_weight_gradient_shifted(pkg, shift):
    """dW_hh = dG^T . h_prev at cfg-B depth: 64 utterances x 1198 steps, h_prev read shifted by one step."""
    _nt_check(pkg.ops, 2048, 512, 1198, 64, shift, True)


_CHUNK_SCRIPT = r"""
import sys, torch
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[1] + "/tests")
import importlib
from conftest import scaled_err
ops = importlib.import_module("end-to-end-asr-pytorch_b200").ops
torch.manual_seed(0)
a = torch.randn(3000, 1000, device="cuda")
w = torch.randn(700, 1000, device="cuda") * 0.05
c = torch.randn(3000, 700, device="cuda")
ref = a.double() @ w.double().t()
errs = [scaled_err(ops.gemm_tn(a, w, w_lo=ops.tf32_residual(w)).cpu().numpy(), ref.cpu().numpy()),
        scaled_err(ops.gemm_nn(a, w.t().contiguous()).cpu().numpy(), ref.cpu().numpy()),
        scaled_err(ops.gemm_nt(a, c, 1000, 700, 3000).cpu().numpy(), (a.double().t() @ c.double()).cpu().numpy())]
print(max(errs))
"""


@pytest.mark.parametrize("chunk", [1, 2, 4])
def test_accumulation_chunk_lengths(pkg, chunk):
    """B200ASR_GEMM_CHUNK is read once per process: each chunk length runs the tn / nn / nt forms in a fresh one."""
    env = dict(os.environ, B200ASR_GEMM_CHUNK=str(chunk))
    r = subprocess.run([sys.executable, "-c", _CHUNK_SCRIPT, ROOT], env=env, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    assert float(r.stdout.strip().splitlines()[-1]) < 3e-6
