"""Static check (no GPU) of the built 3xTF32 GEMM: every gemm3x_kernel instance keeps its fragments and accumulators in
registers (no local memory) and issues wgmma with the A operand from registers (the RS form of the main loop)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "end-to-end-asr-pytorch_b200", "libb200asr.so")
pytestmark = [
    pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="needs cuobjdump"),
    pytest.mark.skipif(not os.path.exists(SO), reason="library not built (run __graft_entry__.build())"),
]


def _per_function(text):
    """{mangled name: body} for cuobjdump's 'Function <name>' sections."""
    out, name = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function\s*:?\s*(\S+?):?\s*$", line)
        if m:
            name = m.group(1)
            out[name] = []
        elif name is not None:
            out[name].append(line)
    return {k: "\n".join(v) for k, v in out.items()}


def test_gemm_kernels_use_no_local_memory():
    text = subprocess.run(["cuobjdump", "--dump-resource-usage", SO], capture_output=True, text=True, check=True).stdout
    funcs = {k: v for k, v in _per_function(text).items() if "gemm3x_kernel" in k}
    assert len(funcs) == 4, sorted(funcs)                      # tn, tn with pre-split B, nn, nt
    for name, body in funcs.items():
        m = re.search(r"LOCAL:(\d+)", body)
        assert m and int(m.group(1)) == 0, (name, body.strip())


def test_gemm_kernels_issue_register_a_wgmma():
    text = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True, check=True).stdout
    funcs = {k: v for k, v in _per_function(text).items() if "gemm3x_kernel" in k}
    assert len(funcs) == 4, sorted(funcs)
    for name, body in funcs.items():
        rs = re.findall(r"HGMMA\.64x128x8\.F32\.TF32 R\d+, R\d+, gdesc", body)
        assert len(rs) >= 12, (name, len(rs))                     # 3 products x 4 k8 steps per K block
        assert not re.search(r"HGMMA\.64x128x8\.F32\.TF32 R\d+, gdesc\[[^]]*\], gdesc", body), name


def test_gemm_kernels_drain_only_at_chunk_boundaries():
    """The main loop keeps one K block's MMAs in flight: the straight-line chunk bodies of length 4, 3, 2 and 1 end in
    one full drain each and wait with one group outstanding inside (3 + 2 + 1 + 0).  Any further full drain would be a
    wait the compiler inserted because it could not track a register operand."""
    text = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True, check=True).stdout
    funcs = {k: v for k, v in _per_function(text).items() if "gemm3x_kernel" in k}
    assert len(funcs) == 4, sorted(funcs)
    for name, body in funcs.items():
        assert len(re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x0", body)) == 4, name
        assert len(re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x1", body)) == 6, name
