"""CPU checks for the GRU encoder layer on the persistent recurrence kernels (tests/test_gpu_gru_encoder.py):

  * the packed 4-slot recurrence (ops.pack_decoder_weights, gate_perm, oracle/gruenc_ref.recurrence, the gradient
    contractions of ops.BiGRUFn and unpack_decoder_grads), all in float64, is nn.GRU in float64 - output, dx and every
    parameter gradient, both directions, with zero-padded ragged utterances;
  * the per-row bound of the GPU tests accepts an fp32 emulation of the kernels' GRU cell and split step products, and
    rejects five planted cell defects by at least 10x;
  * the GRU kernel instances use no more registers or local memory than their LSTM counterparts (so the planner's
    occupancy and cluster queries, asked of the LSTM instances, hold for both cells), and the wgmma ones contain HGMMA.
"""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

import test_gpu_gru_encoder as G
import test_gpu_lstm_variants as V
import test_host_lstm_bounds as LB
from oracle import gruenc_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------- packed layout, float64
def _packed_layer_fp64(ops, params, x, gy, ndir):
    """The layer as BiGRUFn computes it, in float64: packed input projection, recurrence, dG contractions, unpack."""
    B, T, I = x.shape
    H = params[1].shape[1]
    perm = ops.gate_perm(H, "cpu")
    pre, whh, wih = [], [], []
    for d in range(ndir):
        wcat, b = ops.pack_decoder_weights("GRU", *params[4 * d:4 * d + 4])
        wp = wcat[:, :I].index_select(0, perm)
        pre.append((x.reshape(B * T, I) @ wp.t() + b.index_select(0, perm)).view(B, T, H, 4))
        whh.append(wcat[:, I:])
        wih.append(wp)
    out, hst, _, dG = gruenc_ref.recurrence(torch.stack(pre), torch.stack(whh), gy)
    dx = torch.zeros(B * T, I, dtype=torch.float64)
    grads = []
    for d in range(ndir):
        g2 = dG[d].reshape(B * T, 4 * H)                       # unit-major columns
        dx += g2 @ wih[d]
        gm = torch.empty_like(g2)
        gm[:, perm] = g2                                       # gate-major columns (index_copy_ through perm)
        hprev = torch.zeros(B, T, H, dtype=torch.float64)
        if d == 0:
            hprev[:, 1:] = hst[d][:, :-1]
        else:
            hprev[:, :-1] = hst[d][:, 1:]
        dw_ih = gm.t() @ x.reshape(B * T, I)
        dw_hh = gm.t() @ hprev.reshape(B * T, H)
        grads += ops.unpack_decoder_grads("GRU", torch.cat([dw_ih, dw_hh], 1), gm.sum(0), I)
    return out, dx.view(B, T, I), grads


@pytest.mark.parametrize("ndir", [1, 2])
def test_packed_recurrence_equals_nn_gru_fp64(pkg, ndir):
    B, T, I, H = 5, 9, 7, 6
    torch.manual_seed(30 + ndir)
    ref = torch.nn.GRU(I, H, bidirectional=ndir == 2, batch_first=True).double()
    with torch.no_grad():
        for p in ref.parameters():
            p.uniform_(-0.6, 0.6)
    x = torch.randn(B, T, I, dtype=torch.float64)
    x[1, 5:] = 0.0                                             # ragged: zero-padded frames, run over like the reference
    x[3, 2:] = 0.0
    gy = torch.randn(B, T, ndir * H, dtype=torch.float64)
    xr = x.clone().requires_grad_(True)
    yr, _ = ref(xr)
    yr.backward(gy)
    out, dx, grads = _packed_layer_fp64(pkg.ops, [p.detach() for p in ref.parameters()], x, gy, ndir)
    assert float((out - yr.detach()).abs().max()) < 1e-12
    assert float((dx - xr.grad).abs().max()) < 1e-12
    assert len(grads) == len(list(ref.parameters()))
    for g, (name, p) in zip(grads, ref.named_parameters()):
        assert g.shape == p.shape, name
        assert float((g - p.grad).abs().max()) < 1e-12, name


# ------------------------------------------------------------------------------------------- the bound has teeth
DEFECTS = ("b_hn outside the r product", "z and 1 - z swapped", "dh.z carry dropped", "dgh_n without r",
           "h_prev one step late")


def _emulate(pre, whh, dout, dt, fprod, bprod, defect=None):
    """One direction of the GRU recurrence and its BPTT in dtype `dt`, step products by fprod / bprod, in the order of
    the kernels' cell (csrc/rnn_cell.cuh).  pre [B, T, H, 4] (slot 3 = b_hn at h = 0), whh [4H, H]."""
    B, T, H, _ = pre.shape
    pre, w, dout = pre.astype(dt), whh.astype(dt), dout.astype(dt)
    wt = np.ascontiguousarray(w.T)
    h = np.zeros((B, H), dt)
    out, gts = np.zeros((B, T, H), dt), np.zeros((B, T, H, 4), dt)
    for t in range(T):
        hw = fprod(h, wt).astype(dt).reshape(B, 4, H).transpose(0, 2, 1)
        a = pre[:, t] + hw
        r, z = LB._sig(a[..., 0]), LB._sig(a[..., 1])
        if defect == "b_hn outside the r product":
            n = np.tanh(a[..., 2] + pre[:, t, :, 3] + r * hw[..., 3])
        else:
            n = np.tanh(a[..., 2] + r * a[..., 3])
        h = (n - h) * z + h if defect == "z and 1 - z swapped" else (h - n) * z + n
        out[:, t], gts[:, t] = h, np.stack([r, z, n, a[..., 3]], -1)
    dG = np.zeros_like(gts)
    carry = np.zeros((B, H), dt)
    part = np.zeros((B, H), dt)
    lag = 2 if defect == "h_prev one step late" else 1
    for t in range(T - 1, -1, -1):
        r, z, n, ghn = (gts[:, t, :, q] for q in range(4))
        hp = out[:, t - lag] if t >= lag else np.zeros((B, H), dt)
        d = (dout[:, t] + part) + carry
        dgin = d * (1 - z) * (1 - n * n)
        dg = np.stack([dgin * ghn * r * (1 - r), d * (hp - n) * z * (1 - z), dgin,
                       dgin if defect == "dgh_n without r" else dgin * r], -1)
        dG[:, t] = dg
        carry = np.zeros_like(carry) if defect == "dh.z carry dropped" else d * z
        part = bprod(dg.transpose(0, 2, 1).reshape(B, 4 * H), w).astype(dt)
    return out, out, gts, dG


@pytest.mark.parametrize("H,T,wscale,reverse", [(128, 9, 1.0, False), (128, 17, 1.0, True), (256, 9, 3.0, True)])
def test_bound_accepts_the_cell_and_rejects_defects(H, T, wscale, reverse):
    """The reverse direction is the forward recurrence over time-reversed frames (the kernels index h_{t-1} of the
    reverse direction at t + 1); "h_prev one step late" reads the state two steps back in the direction's order."""
    B = 32
    pre, whh, dout = G._inputs(B, T, H, 1, seed=H + T + 50, wscale=wscale)
    if reverse:
        pre, dout = pre.flip(2), dout.flip(1)
    r64 = [t.numpy() for t in gruenc_ref.recurrence(pre, whh, dout, torch.float64)]
    r32 = [t.numpy() for t in gruenc_ref.recurrence(pre, whh, dout, torch.float32)]
    r64 = [r64[0], r64[1][0], r64[2][0], r64[3][0]]
    r32 = [r32[0], r32[1][0], r32[2][0], r32[3][0]]
    pre, whh, dout = pre[0].numpy().astype(np.float64), whh[0].numpy().astype(np.float64), dout.numpy()
    fprod, bprod = LB._split_product, LB._row_scaled(LB._split_product)
    ratios = {name: LB._worst_ratio(_emulate(pre, whh, dout, np.float32, fprod, bprod, name), r64, r32)
              for name in (None,) + DEFECTS}
    print(ratios)
    assert ratios.pop(None) <= 0.5, ratios
    for name, r in ratios.items():
        assert r >= 10.0, (name, r)


# ------------------------------------------------------------------------------------------- kernel resources
def _ptxas(src):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                          "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c", src, "-o", os.devnull],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    res = {}
    for m in re.finditer(r"Compiling entry function '(\S+)'.*?\n.*?\n\s*(\d+) bytes stack frame, (\d+) bytes spill "
                         r"stores, (\d+) bytes spill loads\n.*?Used (\d+) registers", out.stderr):
        res[m.group(1)] = tuple(int(v) for v in m.groups()[1:])
    return res


@pytest.mark.parametrize("src", ["lstm.cu", "lstm_umma.cu"])
def test_gru_instances_use_no_more_than_the_lstm_ones(src):
    """ptxas: each bigru_* step kernel uses at most the registers, stack and spills of the bilstm_* instance with the
    same template arguments."""
    res = _ptxas(os.path.join(ROOT, "end-to-end-asr-pytorch_b200", "csrc", src))
    gru = {k: v for k, v in res.items() if "bigru_" in k}
    assert len(gru) == (4 if src == "lstm.cu" else 9), sorted(res)
    for name, (frame, st, ld, regs) in gru.items():
        ident = re.search(r"bigru_\w*?_kernel", name).group(0)     # mangled as <length><identifier>
        lstm = name.replace("%d%s" % (len(ident), ident), "%d%s" % (len(ident) + 1, ident.replace("bigru", "bilstm")))
        assert lstm in res, (name, lstm)
        lf, ls, ll, lr = res[lstm]
        assert regs <= lr and frame <= lf and st <= ls and ld <= ll, (name, (frame, st, ld, regs), res[lstm])


SO = os.path.join(ROOT, "end-to-end-asr-pytorch_b200", "libb200asr.so")


@pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("c++filt") is None,
                    reason="needs cuobjdump + c++filt")
@pytest.mark.skipif(not os.path.exists(SO), reason="library not built (run __graft_entry__.build())")
def test_gru_wgmma_instances_contain_hgmma():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import sass_mnemonics
    rows = sass_mnemonics.mnemonic_counts(SO)
    fwd = {k: v for k, v in rows.items() if "bigru_fwd_umma_kernel<" in k}
    bwd = {k: v for k, v in rows.items() if "bigru_bwd_umma_kernel<" in k}
    assert len(fwd) == 3 and len(bwd) == 6, sorted(rows)
    for name, r in fwd.items():
        assert r["HGMMA"] >= 4 and r["UBLKCP"] >= 6 and r["SYNCS"] > 0, (name, r)
    for name, r in bwd.items():
        assert r["HGMMA"] >= 4 and r["UBLKCP"] > 0, (name, r)
