"""Scaled dot-product attention, CPU side: the entry points refuse bad arguments before any CUDA call, the Python
limits agree with the library's, the golden dot models' parameter contract, and the shipped kernels use no local
memory."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest
import torch

from conftest import ROOT, load_golden
from oracle.make_golden_dotattn import dotattn_model_cfg

SO = os.path.join(ROOT, "end-to-end-asr-pytorch_b200", "libb200asr.so")
FAKE = ctypes.c_void_p(256)          # never dereferenced: every call below is refused by the argument checks


def _fwd(lib, ptrs, N, R, T, D, E):
    q, k, v, ln, a, c = ptrs
    return lib.b200asr_dotattn_fwd(q, k, v, ln, N, 0.5, R, T, D, E, a, c, None)


def _bwd(lib, ptrs, N, R, T, D, E):
    q, k, v, ln, a, dc, dq, dk = ptrs
    return lib.b200asr_dotattn_bwd_acc(q, k, v, ln, N, 0.5, a, dc, None, R, T, D, E, dq, dk, None)


@pytest.mark.parametrize("which", ["fwd", "bwd"])
def test_null_pointers_and_bad_sizes_are_refused(pkg, which):
    lib = pkg.load_library()
    call, n = (_fwd, 6) if which == "fwd" else (_bwd, 8)
    name = "dotattn_fwd" if which == "fwd" else "dotattn_bwd_acc"
    for i in range(n):
        ptrs = [FAKE] * n
        ptrs[i] = None
        assert call(lib, ptrs, 1, 2, 16, 8, 8) == -1
        assert pkg.lib.last_error() == "%s: null pointer" % name
    ptrs = [FAKE] * n
    for args, msg in [((1, 0, 16, 8, 8), "bad sizes"), ((1, 2, 0, 8, 8), "bad sizes"), ((1, 2, 16, 0, 8), "bad sizes"),
                      ((1, 2, 16, 8, 0), "bad sizes"), ((0, 2, 16, 8, 8), "bad sizes"),
                      ((3, 4, 16, 8, 8), "multiple of N"),
                      ((1, 2, 8193, 8, 8), "frames > 8192"), ((1, 2, 16, 513, 8), "attention dim 513 > 512"),
                      ((1, 2, 16, 8, 6), "multiple of 4"), ((1, 2, 149, 8, 4104), "too large")]:
        assert call(lib, ptrs, *args) == -1, args
        err = pkg.lib.last_error()
        assert err.startswith(name + ":") and msg in err, (args, err)


def test_python_limits_follow_the_library_cluster_rule(pkg):
    """dot_attention_supported equals b200asr_dotattn_supported over a sweep of shapes; a short memory keeps as many
    CTAs as E / CS <= 1024 needs, and only a width the feature split cannot divide is refused."""
    lib = pkg.load_library()
    assert pkg.ops.DOTATTN_MAX_T == 8192
    Ts = [1, 7, 8, 15, 16, 31, 32, 149, 4096, 8191, 8192, 8193]
    Ds = [1, 16, 300, 512, 513]
    Es = [4, 6, 8, 64, 1024, 1028, 2048, 2052, 4096, 4100, 4104, 8192]
    for T in Ts:
        for D in Ds:
            for E in Es:
                py = pkg.ops.dot_attention_supported(T, D, E)
                assert py == bool(lib.b200asr_dotattn_supported(T, D, E)), (T, D, E)
                if not py:       # refused with an argument error, before any CUDA call
                    assert _fwd(lib, [FAKE] * 6, 1, 2, T, D, E) == -1, (T, D, E)
                    assert _bwd(lib, [FAKE] * 8, 1, 2, T, D, E) == -1, (T, D, E)
    assert pkg.ops.dot_attention_supported(4096, 512, 4096)     # 40 s without time reduction, the widest rows
    assert pkg.ops.dot_attention_supported(8, 16, 2048)          # a short memory keeps a 2-CTA cluster: E / CS = 1024
    assert not pkg.ops.dot_attention_supported(8, 16, 4100)      # E % 8 != 0 leaves one CTA: E / CS > 1024


@pytest.mark.parametrize("kind", ["dot1", "dotrep"])
def test_golden_models_have_the_model_state_dict(pkg, kind):
    g = load_golden("model_%s.npz" % kind)
    model = pkg.ASR(g["feat"].shape[-1], g["sd.pre_embed.weight"].shape[0], True, **dotattn_model_cfg(kind))
    ref = {k[3:]: tuple(v.shape) for k, v in g.items() if k.startswith("sd.")}
    assert {k: tuple(v.shape) for k, v in model.state_dict().items()} == ref
    att = model.attention
    assert att.mode == "dot" and not att.v_proj
    assert att.num_head == (1 if kind == "dot1" else 4)
    if kind == "dotrep":           # the repeat reaches another utterance only with more than one utterance per batch
        assert g["feat"].shape[0] >= 3 and len(set(g["encode_len"].tolist())) == g["feat"].shape[0]


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="needs cuobjdump")
@pytest.mark.skipif(not os.path.exists(SO), reason="library not built (run __graft_entry__.build())")
def test_dot_kernels_are_shipped_without_local_memory():
    out = subprocess.run(["cuobjdump", "-res-usage", SO], capture_output=True, text=True, check=True).stdout
    found = {}
    for m in re.finditer(r"Function (\S*dotattn_\w*kernel\S*):\s*\n\s*(REG:.*)", out):
        found[m.group(1)] = dict(kv.split(":") for kv in m.group(2).split())
    names = sorted(found)
    assert len(names) == 3 and sum("dotattn_fwd_kernel" in n for n in names) == 1, names     # fwd + bwd<1>, bwd<2>
    for n, r in found.items():
        assert r["STACK"] == "0" and r["LOCAL"] == "0", (n, r)
